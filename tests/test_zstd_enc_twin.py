"""The CPU twin of the zstd encoder's entropy stage (oracle/zstd_enc_twin.c, through _zenc.framed_b200) on its own:
the frames it writes decode to the source through the oracle and through libzstd, keep the encoder's mode rules and
carry the intended Huffman code; every case of the entropy-edge corpus (_zentcorpus) reaches its edge and its
knock-out does not; the schedule model's constants are the kernel's.  The GPU streams are held to these frames byte for
byte by the GPU tests."""
import numpy as np
import pytest

import _oracle as o
import _pipecorpus as pc
import _searchcorpus as sc
import _zcorpus as zco
import _zenc as ze
import _zentcorpus as zc
import _zentsched as zs
import zstdmt_b200 as z
from test_gpu_zstd_encoder import check_huffman, check_modes, edge_windows

CASES = {c.name: c for c in zc.cases()}


def frames_ok(src, chunk, level, chunk_bytes=None):
    """framed_b200 of src: decoded by the oracle and by libzstd (frame by frame) to each chunk, mode rules, Huffman
    lengths.  Returns the twin's (chunk, block, BlockTrace) list."""
    blocks = []
    framed = ze.framed_b200(src, chunk, level, chunk_bytes, blocks)
    parts = ze.chunks(src, chunk, chunk_bytes)
    frames = o.mt_frames(framed)
    assert len(frames) == len(parts)
    for f, content in zip(frames, parts):
        tr = o.zstd_trace(f)
        assert np.array_equal(tr.content, content)
        check_modes(tr)
        for b in range(len(tr.blk)):
            if tr.blk[b, o.ZT["type"]] == 2:
                check_huffman(tr, b, _Rep())
        assert np.array_equal(zco.libzstd_decompress(f, max(content.size, 1)), content)
    whole = np.concatenate(parts) if parts else src
    rc, back = o.orc_decode(o.CODEC_ZSTD, framed, max(whole.size, 1))
    assert rc == 0 and np.array_equal(back, whole)
    return blocks


class _Rep:
    huf = 0


def _gen(kind, n, seed):
    return z.gen_stream(kind, n, 1 << 20, first=seed)


@pytest.mark.parametrize("level", [3, 9])
@pytest.mark.parametrize("kind", ["text", "mix", "zeros", "random"])
def test_twin_frames_of_generated_input(kind, level):
    k = {"text": z.GEN_TEXT, "mix": z.GEN_MIX, "zeros": z.GEN_ZEROS, "random": z.GEN_RANDOM}[kind]
    src = _gen(k, 300000 + level, 3)
    blocks = frames_ok(src, 1 << 17, level)
    modes = {(t.lit_mode, bool(t.raw_reason)) for _, _, t in blocks}
    if kind == "random":
        assert modes == {(0, True)}
    if kind == "zeros":
        assert (1, False) in modes
    if kind in ("text", "mix"):
        assert (2, False) in modes


@pytest.mark.parametrize("name", sorted(CASES))
def test_corpus_case_frames(name):
    c = CASES[name]
    src, chunk, cb = c.built()
    for level in sorted({3, c.level}):
        frames_ok(src, chunk, level, cb)


@pytest.mark.parametrize("name", sorted(CASES))
def test_corpus_case_reaches_its_edge_and_its_knockout_does_not(name):
    c = CASES[name]
    assert c.reaches(c.k), c.doc
    assert not c.reaches(c.knock()), ("knocked out, still reached", c.doc)


def test_edge_windows_and_corpora():
    """The level-3 edge windows of test_gpu_zstd_encoder, the schedule corpus of the level-3 / LZ4 tile pipeline and the
    zstd cases of the search corpus at their levels."""
    for name, wins in edge_windows().items():
        frames_ok(np.concatenate(wins), 1 << 20, 3)
    for b in pc.BUILDERS:
        src, chunk, marks, _ = b()
        parts = pc.parts(src, chunk, marks)
        if chunk is None:
            frames_ok(np.concatenate(parts), max(p.size for p in parts), 3, [p.size for p in parts])
        else:
            frames_ok(src, chunk, 3)
    for case in sc.cases():
        if case.codec == "zstd":
            for level in case.levels:
                frames_ok(case.src, case.chunk, level, case.chunk_bytes)


def test_events_name_the_block_fields():
    """On the tokens window (thousands of short sequences per sub-block) the model's repair loop runs for several rounds
    and still ends on the serial chain's states (chain_model asserts it); its Huffman runs tile each stream."""
    win = edge_windows()["tokens"][0]
    evs = [ev for _, ev in zs.chunk_events(win, 3)]
    assert max(ev["nseq"] for ev in evs) > 3000
    assert any(ev.get("repair_rounds_ML", 0) >= 2 for ev in evs)
    assert all(ev["huf_shared_words"] > 0 for ev in evs if ev["lit_mode"] == 2)


def test_model_constants_match_the_kernel():
    """The schedule model's and the twin's constants are the #defines of zstd_entropy.cuh."""
    k = zs.kernel_constants()
    assert (zs.Z_WARM, zs.Z_BITWORDS, zs.Z_HUF_MAXBITS, zs.Z_MAXSEQ, zs.Z_MAXLIT) == \
           (k["Z_WARM"], k["Z_BITWORDS"], k["Z_HUF_MAXBITS"], k["Z_MAXSEQ"], k["Z_MAXLIT"])
    assert ze.BITBUF == 4 * k["Z_BITWORDS"]
    import os
    import re
    twin = open(os.path.join(o.ROOT, "oracle", "zstd_enc_twin.c")).read()
    got = {m.group(1): eval(re.sub(r"(\d+)u\b", r"\1", m.group(2).split("/*")[0]))
           for m in re.finditer(r"^#define\s+T_(BITWORDS|HUF_MAXBITS|MAXSEQ|MAXLIT)\s+(.+)$", twin, re.M)}
    assert got == {"BITWORDS": k["Z_BITWORDS"], "HUF_MAXBITS": k["Z_HUF_MAXBITS"], "MAXSEQ": k["Z_MAXSEQ"], "MAXLIT": k["Z_MAXLIT"]}
