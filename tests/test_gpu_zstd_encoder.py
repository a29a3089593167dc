"""The GPU zstd encoder (zstd_blocks_kernel + z_encode_block) held block by block to what it means to produce
(pytest -m gpu).  Every frame is traced by the oracle (orc_zstd_trace) and checked against:
  (a) the parse: each compressed sub-block's sequences are the CPU twin's LZ4 sequences whose matches start inside it,
      and the sub-blocks are cut where _zenc.sub_blocks says;
  (b) the Huffman code: the traced code lengths are those of _zenc.huf_lengths on the block's literal histogram;
  (c) the mode rules of the default build (see check_modes);
  (d) the round trip: oracle, libzstd (both paths, when oracle/_ref exists) and the GPU decoder;
  (e) the bytes: the framed stream equals _zenc.framed_b200 (the entropy stage's CPU twin on the twin parse).
Inputs are built here with fixed seeds; each edge case asserts from the trace that it reached its edge."""
import numpy as np
import pytest

import _oracle as o
import _zenc as ze
import zstdmt_b200 as z
from _zxmodel import ML_BASE

pytestmark = pytest.mark.gpu
ZT = o.ZT
W = ze.WINDOW
Z_BITBUF = ze.BITBUF             # the entropy stage's bit buffer (Z_BITWORDS words)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


# ------------------------------------------------------------------------------------------------- compress + trace
def gpu_compress(torch, src, chunk, chunk_bytes=None):
    """zmt_zstd_compress_device.  chunk_bytes: explicit per-chunk sizes, chunk c read from src[c * chunk:]."""
    L = z.lib()
    n = int(src.size)
    if chunk_bytes is None:
        nch = L.zmt_chunk_count(n, chunk); d_cb = None
    else:
        nch = len(chunk_bytes); d_cb = torch.from_numpy(np.asarray(chunk_bytes, np.int32)).cuda()
    d_in = torch.from_numpy(src).cuda() if n else torch.empty(1, dtype=torch.uint8, device="cuda")
    work = torch.empty(L.zmt_zstdc_workspace_bytes(nch, chunk), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_zstdc_out_bound(nch, chunk), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(nch + 1, dtype=torch.int64, device="cuda")
    rc = L.zmt_zstd_compress_device(d_in.data_ptr(), n, chunk, d_cb.data_ptr() if d_cb is not None else None, nch,
                                    work.data_ptr(), out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy()


def chunks_of(src, chunk, chunk_bytes):
    if chunk_bytes is None:
        return [src[i: i + chunk] for i in range(0, max(src.size, 1), chunk)]
    return [src[c * chunk: c * chunk + int(b)] for c, b in enumerate(chunk_bytes)]


class Report:
    def __init__(self):
        self.sub = self.raw = self.huf = 0
        self.blocks = []                 # (trace, block index, start in the frame's content) of every non-empty block
        self.twin = []                   # (chunk, block, _zenc.BlockTrace) of every block the twin wrote
        self.raw_by = {}                 # raw blocks by reason, from the twin's traces (_zenc.raw_counts)

    @property
    def raw_bitbuf(self):
        return self.raw_by.get("bitbuf", 0)

    def share(self):
        return self.raw_bitbuf / max(1, self.sub)


def check(torch, src, chunk=1 << 20, chunk_bytes=None):
    """Compress on the GPU, trace every frame and check (a)-(e).  Returns the Report with every compressed block."""
    framed = gpu_compress(torch, src, chunk, chunk_bytes)
    frames = o.mt_frames(framed)
    parts = chunks_of(src, chunk, chunk_bytes)
    assert len(frames) == len(parts)
    rep = Report()
    rep.twin = ze.assert_twin(framed, src, chunk, 3, chunk_bytes)
    rep.raw_by = ze.raw_counts(rep.twin)
    for f, content in zip(frames, parts):
        tr = o.zstd_trace(f)
        assert np.array_equal(tr.content, content)
        check_modes(tr)
        pos = 0
        for b in range(len(tr.blk)):
            regen = int(tr.blk[b, ZT["regen"]])
            if regen:
                rep.blocks.append((tr, b, pos))
            pos += regen
        check_windows(tr, content, rep)
    check_roundtrip(torch, framed, src if chunk_bytes is None else np.concatenate(parts) if parts else src)
    return rep


def check_modes(tr):
    """(c) the mode rules of the encoder."""
    typ, last, regen, bsize = tr.col("type"), tr.col("last"), tr.col("regen"), tr.col("bsize")
    assert set(typ.tolist()) <= {0, 2}                              # raw or compressed blocks only
    assert list(last) == [0] * (len(last) - 1) + [1]                 # only the last block is flagged last
    assert (regen <= 128 * 1024).all() and (bsize <= 128 * 1024).all()
    for b in np.flatnonzero(typ == 2):
        r = tr.blk[b]
        lt, nlit = int(r[ZT["lit_type"]]), int(r[ZT["lit_regen"]])
        lits = tr.block_lits(b)
        assert bsize[b] < regen[b]                                   # a compressed block is smaller than its content
        ndist = np.unique(lits).size
        assert (lt == 1) == (ndist == 1), (b, lt, ndist)             # RLE literals iff one distinct byte
        assert lt in (0, 1, 2)                                       # every block carries its own tree
        if lt == 2:
            assert nlit >= 64 and r[ZT["lit_streams"]] == 4
            comp = int(r[ZT["lit_comp"]])
            want = 3 if nlit < 1024 and comp < 1024 else 4 if nlit < 16384 and comp < 16384 else 5
            assert r[ZT["lit_hdr"]] == want, (b, nlit, comp)
            maxsym = int(lits.max())
            assert r[ZT["nweights"]] == maxsym                        # symbols 0 .. maxsym-1 listed, the last implied
            assert (r[ZT["tree_form"]] == 0) == (maxsym <= 128)        # direct weights iff they can express the alphabet
            assert r[ZT["maxbits"]] <= 11
        else:
            assert r[ZT["lit_hdr"]] == (1 if nlit < 32 else 2 if nlit < 4096 else 3)
        nseq = int(r[ZT["nseq"]])
        assert r[ZT["nseq_bytes"]] == (1 if nseq < 128 else 2)
        if nseq:
            assert r[ZT["modes"]] == 0                               # predefined tables for LL, OF and ML
            assert (tr.block_seqs(b)[:, 1] > 3).all()                # explicit offsets only: no repeat codes


def check_windows(tr, content, rep):
    """(a) and (b) for one frame: walk its 64 KiB windows."""
    starts = np.concatenate([[0], np.cumsum(tr.col("regen"))])
    for w0 in range(0, content.size, W):
        win = content[w0: w0 + W]
        model = ze.window_model(win)
        sel = [b for b in range(len(tr.blk)) if w0 <= starts[b] < w0 + W and tr.blk[b, ZT["regen"]]]
        got = [(int(starts[b]) - w0, int(starts[b + 1]) - w0) for b in sel]
        assert got == [(a, e) for a, e, _ in model], ("sub-block cut differs from the twin", w0, got, [(a, e) for a, e, _ in model])
        for b, (a, e, mseq) in zip(sel, model):
            rep.sub += 1
            if tr.blk[b, ZT["type"]] == 0:
                rep.raw += 1
                continue
            q = tr.block_seqs(b).astype(np.int64)
            if len(q):
                ends = a + np.cumsum(q[:, 0] + q[:, 2])
                mine = np.stack([ends - q[:, 2], q[:, 1] - 3, q[:, 2]], axis=1)
            else:
                mine = np.zeros((0, 3), np.int64)
            assert np.array_equal(mine, mseq), ("parse differs from the twin", w0, a, e)
            check_huffman(tr, b, rep)


def check_huffman(tr, b, rep):
    """(b) the traced code is the intended one: lengths maxbits + 1 - weight equal the twin's on the literal histogram."""
    if tr.blk[b, ZT["lit_type"]] != 2:
        return
    rep.huf += 1
    hist = np.bincount(tr.block_lits(b), minlength=256)
    want, wmax = ze.huf_lengths(hist)
    mb = int(tr.blk[b, ZT["maxbits"]])
    w = tr.weights[b].astype(np.int64)
    got = {int(s): mb + 1 - int(w[s]) for s in np.flatnonzero(w)}
    assert mb == wmax and got == want, ("Huffman lengths differ from the twin", b)
    assert ze.kraft(got, mb) == 1 << mb


def check_roundtrip(torch, framed, src):
    """(d) libzstd on its single- and multi-thread paths, the oracle, our GPU decoder."""
    n = int(src.size)
    rc, back = o.orc_decode(o.CODEC_ZSTD, framed, n)
    assert rc == 0 and np.array_equal(back, src)
    if o.have_ref():
        for T in (1, 3):
            rc, back, _ = o.ref_decompress(o.CODEC_ZSTD, framed, n, threads=T)
            assert rc == 0 and np.array_equal(back, src)
    dec = z.ZstdDeviceDecompressor(framed)
    out, status = dec.run(torch.from_numpy(np.ascontiguousarray(framed)).cuda())
    torch.cuda.synchronize()
    assert not status.cpu().numpy()[: dec.n].any() and np.array_equal(out[: dec.out_total].cpu().numpy(), src)


# ------------------------------------------------------------------------------------------------- inputs
def rnd(rng, n, hi=256):
    return rng.integers(0, hi, n, dtype=np.uint8) if n else np.zeros(0, np.uint8)


RUN = 5000                       # zeros opening each sub-block of the literal-alphabet windows


def with_runs(fill):
    """Each 16 KiB sub-block: RUN zeros (one match, where the block is cut), then fill(k, 16384 - RUN) literals.  The
    literal sections stay small enough for the Huffman bit stream to fit the entropy stage's buffer."""
    return np.concatenate([np.concatenate([np.zeros(RUN, np.uint8), fill(k, ze.SUB - RUN)]) for k in range(W // ze.SUB)])


def fib_window(rng):
    """Groups (x, x', counter high, counter low) with no repeated 4-gram, so every byte is a literal; the x carry
    Fibonacci counts (1, 1, 2, 3, 5, ...) over 17 symbols: the unlimited Huffman tree is deeper than 11."""
    fib = [1, 1]
    while len(fib) < 17:
        fib.append(fib[-1] + fib[-2])

    def fill(k, n):
        g = np.arange(k * n // 4, (k + 1) * n // 4)
        x = np.repeat(np.arange(1, 18, dtype=np.uint8), fib)
        x = rng.permutation(np.concatenate([x, np.full(2 * g.size - x.size, 17, np.uint8)]))
        return np.stack([x[0::2], x[1::2], (32 + (g >> 7)).astype(np.uint8), (128 + (g & 127)).astype(np.uint8)], axis=1).reshape(-1)
    return with_runs(fill)


def alphabet_window(rng, top, skew=False, run=True):
    """Random literals over 0..top, all of them present in every sub-block; skew: the lower half four times as frequent.
    run=False: one 2000-byte match per sub-block only, so the literal section outgrows the Huffman bit buffer."""
    p = np.ones(top + 1)
    if skew:
        p[: (top + 1) // 2] = 4

    def fill(k, n):
        x = rng.choice(top + 1, n, p=p / p.sum()).astype(np.uint8)
        x[100] = top
        return x
    if run:
        return with_runs(fill)
    return np.concatenate([np.concatenate([np.zeros(2000, np.uint8), fill(k, ze.SUB - 2000)]) for k in range(W // ze.SUB)])


def binary_prefix(rng, n):
    """n bytes over {0, 1} in which no 4-gram equals the one 1..4 positions before it: in the first 1024 positions of a
    window (no hash-table candidates yet) every one of them is a literal."""
    s = []
    while len(s) < n:
        for b in rng.permutation(2):
            s.append(int(b))
            i = len(s) - 4
            if i < 0 or all(s[i: i + 4] != s[i - d: i - d + 4] for d in range(1, 5) if i - d >= 0):
                break
            s.pop()
        else:
            s = s[:-8] if len(s) > 8 else []
    return np.array(s, np.uint8)


def binary_window(rng, nbin):
    """Binary literals, a run of zeros (a match), a 1, then zeros to the window end (a second match, pending until the
    window's last block, whose literals are RLE).  The first block: nbin + 2 or so literals over {0, 1} and one match."""
    return np.concatenate([binary_prefix(rng, nbin), np.zeros(200, np.uint8), np.ones(1, np.uint8),
                           np.zeros(W - nbin - 201, np.uint8)])


def tuned(make, target, lo, hi, what):
    """make(k) for the k in [lo, hi) whose twin model has a sub-block with what(...) == target."""
    for k in range(lo, hi):
        win = make(k)
        for a, e, s in ze.window_model(win):
            if what(win, a, e, s) == target:
                return win
    raise AssertionError("no input reaches %r" % (target,))


def nlit_of(win, a, e, s):
    return (e - a) - (int(s[:, 2].sum()) if len(s) else 0)


def runs_window(rng, n1, n2):
    """Random bytes with n1 runs of 8 equal bytes in the first 16 KiB and n2 in the second: one sequence per run."""
    x = rnd(rng, W)
    for k in range(n1):
        x[200 + k * 120: 208 + k * 120] = x[199 + k * 120] ^ 0x55
    for k in range(n2):
        x[ze.SUB + 200 + k * 120: ze.SUB + 208 + k * 120] = x[ze.SUB + 199 + k * 120] ^ 0x55
    return x


def period4(rng, L):
    """A guard byte, a random 4-byte pattern, then L more bytes of it (one match of offset 4 and length L), a breaker."""
    p = rnd(rng, 4)
    while len(set(p.tolist())) < 4:
        p = rnd(rng, 4)
    body = np.resize(p, 4 + L)
    brk = np.uint8((int(p[L % 4]) + 1) % 256)
    return np.concatenate([np.array([p[3] ^ 0x80, *body, brk], np.uint8), rnd(rng, 7)])


def ml_windows(rng):
    """Matches of every length on either side of each ML code boundary (4 .. 32771), packed into windows."""
    lens = sorted({v for b in ML_BASE[2:52] for v in (b - 1, b)})
    segs = [period4(rng, L) for L in lens]
    return pack(rng, segs)


def offset_windows(rng):
    """Random 12-byte strings repeated at distance d, zeros in between: the copy is a match of offset d.  The zeros put
    one 4-gram in the hash table, so the string's slot survives the distance; each string sits 16 bytes before a
    1024-position round boundary, so its copy lies in a later round (the table only holds earlier rounds)."""
    ds = sorted({v for k in range(4, 16) for v in ((1 << k) - 4, (1 << k) - 3)} | {32765})
    wins, win, pos = [], None, 0
    for d in ds:
        if win is None or pos + d + 40 > W - 16:
            win = np.zeros(W, np.uint8); wins.append(win); pos = 1008
        s = rnd(rng, 12)
        win[pos: pos + 12] = s; win[pos + d: pos + d + 12] = s; win[pos + d + 12: pos + d + 20] = rnd(rng, 8)
        pos = (pos + d + 40 + 1023) // 1024 * 1024 + 1008
    last = np.zeros(W, np.uint8); s = rnd(rng, 12)                   # the largest offset a window allows
    last[8:20] = s; last[65508:65520] = s; last[65520:65528] = rnd(rng, 8)
    return wins + [last]


def pack(rng, segs):
    """Segments laid out into whole 64 KiB windows (a segment never crosses a window), random filler between."""
    wins, cur = [], []
    for s in sorted(segs, key=len, reverse=True):
        placed = False
        for wl in wins + [cur]:
            if sum(len(x) for x in wl) + len(s) + 16 <= W - 16:
                wl.append(rnd(rng, 16)); wl.append(s); placed = True
                break
        if not placed:
            cur = [rnd(rng, 16), s]
            wins.append(cur)
    out = []
    for wl in wins:
        x = np.concatenate(wl)
        out.append(np.concatenate([x, rnd(rng, W - x.size)]))
    return out


def token_window(rng, ntok=60):
    """Concatenated short tokens from a dictionary: sub-blocks of ~4000 short sequences."""
    toks = [rnd(rng, int(rng.integers(4, 6))) for _ in range(ntok)]
    out, size = [], 0
    while size < W:
        t = toks[int(rng.integers(0, ntok))]
        out.append(t); size += t.size
    return np.concatenate(out)[:W]


def lit16k_window(rng, nlit):
    """One long match pending from byte 1, then nlit literals: groups (x, x', counter high, counter low) with no repeated
    4-gram and about 4 bits of entropy per byte.  No later match replaces the pending one, so no sub-block is cut before
    the window ends, and the final block carries all nlit literals, Huffman-coded within the bit buffer."""
    g = np.arange((nlit + 3) // 4)
    x = rnd(rng, 2 * g.size, 4)
    lits = np.stack([x[0::2], x[1::2], (64 + (g >> 8)).astype(np.uint8), (g & 255).astype(np.uint8)], axis=1).reshape(-1)
    return np.concatenate([np.full(41, 200, np.uint8), lits[:nlit]])


def edge_windows():
    """name -> list of windows, each 64 KiB."""
    rng = np.random.default_rng(2024)
    E = {}
    E["fibonacci"] = [fib_window(rng)]
    for top in (127, 128, 129):
        E["maxsym%d" % top] = [alphabet_window(rng, top)]
    E["maxsym255_all256"] = [alphabet_window(rng, 255, skew=True)]
    E["lit_bitbuf"] = [alphabet_window(rng, 127, run=False)]
    for k in (63, 64, 1023, 1024):
        E["nlit%d" % k] = [tuned(lambda s, k=k: binary_window(np.random.default_rng(s), k + s % 4 - 2), k, 0, 64, nlit_of)]
    E["nseq127"] = [tuned(lambda k: runs_window(np.random.default_rng(5), k, k + 1), 127, 124, 131, lambda w, a, e, s: len(s))]
    E["nseq128"] = [tuned(lambda k: runs_window(np.random.default_rng(6), k, k + 1), 128, 124, 131, lambda w, a, e, s: len(s))]
    E["ml_codes"] = ml_windows(rng)
    E["offsets"] = offset_windows(rng)
    E["tokens"] = [token_window(rng)]
    E["zeros"] = [np.zeros(W, np.uint8)]
    return E


_EDGE = None


def edges():
    global _EDGE
    if _EDGE is None:
        _EDGE = edge_windows()
    return _EDGE


def entropy_edge_windows():
    """The inputs of the entropy-edge corpus (_zentcorpus) that fit one window, each zero-padded to 64 KiB."""
    import _zentcorpus as zc
    out = []
    for c in zc.cases():
        src = c.built()[0]
        if src.size <= W:
            out.append(np.concatenate([src, np.zeros(W - src.size, np.uint8)]))
    return out


def huff_blocks(rep):
    return [(tr, b) for tr, b, _ in rep.blocks if tr.blk[b, ZT["type"]] == 2 and tr.blk[b, ZT["lit_type"]] == 2]


def reached(name, rep):
    """Assert from the trace that the windows of `name` reached their edge."""
    H = huff_blocks(rep)
    comp = [(tr, b) for tr, b, _ in rep.blocks if tr.blk[b, ZT["type"]] == 2]
    if name == "fibonacci":                                          # the length limiter ran
        assert any(ze.huf_lengths(np.bincount(tr.block_lits(b), minlength=256), limit=False)[1] > 11
                   and tr.blk[b, ZT["maxbits"]] == 11 for tr, b in H)
    elif name.startswith("maxsym"):
        top = 255 if name.startswith("maxsym255") else int(name[6:])
        hit = [(tr, b) for tr, b in H if tr.blk[b, ZT["nweights"]] == top]
        assert hit
        for tr, b in hit:
            assert tr.blk[b, ZT["tree_form"]] == (1 if top > 128 else 0)
        if top == 255:
            assert any(np.unique(tr.block_lits(b)).size == 256 for tr, b in hit)      # 255 FSE-coded weights
    elif name in ("nlit63", "nlit64"):                              # the Huffman threshold, on a 2-symbol alphabet
        k = int(name[4:])
        hit = [(tr, b) for tr, b in comp if tr.blk[b, ZT["lit_regen"]] == k and np.unique(tr.block_lits(b)).size == 2]
        assert hit and all(tr.blk[b, ZT["lit_type"]] == (2 if k >= 64 else 0) for tr, b in hit)
    elif name in ("nlit1023", "nlit1024"):                          # the 3- / 4-byte Huffman literal header
        k = int(name[4:])
        hit = [(tr, b) for tr, b in H if tr.blk[b, ZT["lit_regen"]] == k]
        assert hit and all(tr.blk[b, ZT["lit_hdr"]] == (3 if k < 1024 else 4) for tr, b in hit)
        assert any(tr.blk[b, ZT["lit_type"]] == 1 for tr, b in comp)                  # the zeros after it: RLE literals
    elif name in ("nseq127", "nseq128"):                            # the 1- / 2-byte nbSeq
        k = int(name[4:])
        hit = [(tr, b) for tr, b in comp if tr.blk[b, ZT["nseq"]] == k]
        assert hit and all(tr.blk[b, ZT["nseq_bytes"]] == (1 if k < 128 else 2) for tr, b in hit)
    elif name == "ml_codes":                                        # both sides of every ML code boundary
        ml = set()
        for tr, b in comp:
            ml |= set(tr.block_seqs(b)[:, 2].tolist())
        want = {v for bb in ML_BASE[2:51] for v in (bb - 1, bb)} - {4} | {32770}
        assert want <= ml, sorted(want - ml)                       # code 51 (32771 and up): the zeros window
        # a match pending across a sub-block cut: a block that starts with a match reaching past the next 16 KiB mark
        assert any(pos % W % ze.SUB and tr.blk[b, ZT["nseq"]] > 0 and tr.block_seqs(b)[0, 0] == 0
                   and pos % W + int(tr.block_seqs(b)[0, 2]) > (pos % W // ze.SUB + 1) * ze.SUB
                   for tr, b, pos in rep.blocks if tr.blk[b, ZT["type"]] == 2)
    elif name == "offsets":                                         # Offset_Value = off + 3 on both sides of 2^k
        of = set()
        for tr, b in comp:
            of |= set((tr.block_seqs(b)[:, 1]).tolist())
        want = {v for k in range(7, 16) for v in ((1 << k) - 1, 1 << k)} | {65503}
        assert want <= of, sorted(want - of)
    elif name == "lit_bitbuf":                                      # Huffman would pay, but its bits overflow the buffer
        hit = []
        for tr, b in comp:
            lits = tr.block_lits(b)
            if tr.blk[b, ZT["lit_type"]] == 0 and lits.size >= 64:
                h = np.bincount(lits, minlength=256); ln, _ = ze.huf_lengths(h)
                est = (sum(int(h[s]) * x for s, x in ln.items()) + 7) // 8 + 4 + 1 + (int(lits.max()) + 1) // 2 + 6
                if est < lits.size and est + 64 > Z_BITBUF:
                    hit.append(b)
        assert hit
    elif name == "tokens":                                          # sub-blocks of thousands of short sequences
        assert max(int(tr.blk[b, ZT["nseq"]]) for tr, b in comp) >= 3000
    elif name == "zeros":
        assert any(tr.blk[b, ZT["lit_type"]] == 1 for tr, b in comp)
        assert any(int(tr.block_seqs(b)[:, 2].max()) > 65000 for tr, b in comp if tr.blk[b, ZT["nseq"]] > 0)


# ------------------------------------------------------------------------------------------------- tests
EDGE_NAMES = ["fibonacci", "maxsym127", "maxsym128", "maxsym129", "maxsym255_all256", "lit_bitbuf", "nlit63", "nlit64", "nlit1023",
              "nlit1024", "nseq127", "nseq128", "ml_codes", "offsets", "tokens", "zeros"]


@pytest.mark.parametrize("name", EDGE_NAMES)
def test_encoder_edge_windows(torch, name, capsys):
    src = np.concatenate(edges()[name])
    rep = check(torch, src)
    reached(name, rep)
    if name == "tokens":
        with capsys.disabled():
            print("\n[zstd encoder] tokens: %d of %d sub-blocks stored raw: %d not smaller than their content, %d (%.1f %%) because "
                  "the sequence bits overflow the %d-byte bit buffer" % (rep.raw, rep.sub, rep.raw_by["size"], rep.raw_bitbuf,
                                                                          100 * rep.share(), Z_BITBUF))


def test_encoder_literal_sections_around_16k(torch):
    """Literal sections of 16383 / 16384 / 16385 bytes (4- and 5-byte Huffman headers), in windows that end their chunk."""
    rng = np.random.default_rng(16)
    sizes = [16383, 16384, 16385]
    chunk = W
    wins = [lit16k_window(rng, k) for k in sizes]
    src = np.zeros(chunk * len(wins), np.uint8)
    for i, w in enumerate(wins):
        src[i * chunk: i * chunk + w.size] = w
    rep = check(torch, src, chunk, [w.size for w in wins])
    H = huff_blocks(rep)
    for k in sizes:
        hit = [(tr, b) for tr, b in H if tr.blk[b, ZT["lit_regen"]] == k]
        assert hit and all(tr.blk[b, ZT["lit_hdr"]] == (4 if k < 16384 else 5) for tr, b in hit), k


def test_encoder_ragged_chunks_and_short_windows(torch):
    """Explicit chunk sizes: windows of 1..12 trailing bytes, an empty chunk, ragged sizes, raw literal headers."""
    rng = np.random.default_rng(12)
    chunk = 3 * W
    sizes = [W + k for k in range(1, 13)] + [0, 1, 12, 31, 32, 2 * W + 4095, 2 * W + 4096, 3 * W, 100003 - W]
    src = np.zeros(chunk * len(sizes), np.uint8)
    for c, k in enumerate(sizes):
        src[c * chunk: c * chunk + k] = z.gen_stream(z.GEN_MIX, k, 1 << 20, first=2 + c % 6)
    rep = check(torch, src, chunk, sizes)
    assert rep.sub > len(sizes)


def test_encoder_state_does_not_leak_across_windows_of_one_cta(torch, capsys):
    """About 72 MiB: more windows than the persistent grid has CTAs, so CTA c also encodes window c + grid.  The edge
    windows (and the entropy-edge corpus's level-3 inputs) are laid out so that each of those CTAs meets two different
    kinds in turn; the rest is the Silesia-like mix."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    grid = min(sm * 8, 132 * 8)
    E = edges()
    kinds = [w for name in EDGE_NAMES for w in E[name]] + entropy_edge_windows()
    nwin = grid + 96
    src = z.gen_stream(z.GEN_MIX, nwin * W, 1 << 20, first=1)
    for i in range(96):
        src[i * W: (i + 1) * W] = kinds[i % len(kinds)]
        src[(i + grid) * W: (i + grid + 1) * W] = kinds[(i + 1 + i // len(kinds)) % len(kinds)]
    rep = check(torch, src)
    with capsys.disabled():
        print("\n[zstd encoder] %.1f MiB, grid %d: %d sub-blocks, %d Huffman, %d raw: %d not smaller than their content, %d "
              "(%.2f %%) because the sequence bits overflow the bit buffer" % (src.size / 2**20, grid, rep.sub, rep.huf, rep.raw,
                                                                              rep.raw_by["size"], rep.raw_bitbuf, 100 * rep.share()))
    assert src.size > grid * W
