"""The CPU twin of the LZ4 level 10-12 class (oracle/chain_twin.c) against the rule restated in Python
(tests/_lz4hc.py), the frames it writes, and the LZ4 level table of LZ4MT_createCCtx.  No GPU involved."""
import os
import subprocess
import sys

import numpy as np
import pytest

import _lz4hc as hc
import _oracle as o
import zstdmt_b200 as z


def inputs():
    rng = np.random.default_rng(2025)
    per = lambda p, n: np.resize(rng.integers(0, 256, p, dtype=np.uint8), n)
    yield "text", z.gen_stream(z.GEN_TEXT, 100 << 10, 1 << 20)
    yield "mix", z.gen_stream(z.GEN_MIX, 70000, 1 << 20, first=2)
    yield "zeros", np.zeros(20000, np.uint8)
    yield "random", rng.integers(0, 256, 30000, dtype=np.uint8)
    for p in (1, 2, 3, 4):
        yield "period%d" % p, per(p, 9000 + p)
    yield "small-alphabet", rng.integers(0, 3, 25000, dtype=np.uint8)
    yield "empty", np.zeros(0, np.uint8)
    yield "one", np.array([9], np.uint8)
    yield "twelve", per(2, 12)
    yield "thirteen", per(2, 13)


DATA = dict(inputs())
CASES = [(name, lv, W, B) for name in DATA for lv in hc.LEVELS for W, B in ((0, 0), (4096, 1024), (700, 3000))]


@pytest.mark.parametrize("name,level,W,B", CASES)
def test_twin_equals_restatement_and_replays(name, level, W, B):
    src = DATA[name]
    if name == "text" and not W and level > 10:
        src = src[: 40 << 10]                          # the restatement walks up to 256 candidates per position in Python
    want = hc.sequences(src, level, W=W or None, block=B or hc.BLOCK)
    got = hc.twin_sequences(src, level, W, B)
    assert len(got) == len(want)
    for b, (g, w) in enumerate(zip(got, want)):
        assert [tuple(x) for x in g.tolist()] == w, (name, level, W, B, b)
    assert hc.replay(src, want, B or hc.BLOCK) == src.tobytes()
    if W:
        assert all(off <= W for seqs in want for _, off, _ in seqs)


@pytest.mark.parametrize("name", ["mix", "zeros", "random", "period3", "empty", "one", "thirteen"])
def test_twin_frame_equals_restated_frame(name):
    src = DATA[name]
    for level in hc.LEVELS:
        framed = hc.twin_compress(src, 1 << 20, level)
        assert framed.tobytes() == hc.frame(src, level, lambda b: o.xxh32(np.frombuffer(b, np.uint8) if b else np.zeros(0, np.uint8)))


def corpus():
    rng = np.random.default_rng(7)
    parts = [z.gen_stream(z.GEN_TEXT, 300000, 1 << 20), z.gen_stream(z.GEN_MIX, 200000, 1 << 20, first=5), np.zeros(70000, np.uint8),
             rng.integers(0, 256, 70000, dtype=np.uint8), np.resize(rng.integers(0, 256, 3, dtype=np.uint8), 66000)]
    return np.concatenate(parts)


@pytest.mark.parametrize("level", hc.LEVELS)
def test_twin_frames_are_restored_and_well_formed(level):
    src = corpus()
    chunk = 200000                                      # not a multiple of 64 KiB: every chunk ends in a short block
    framed = hc.twin_compress(src, chunk, level)
    parts = [src[i: i + chunk] for i in range(0, src.size, chunk)]
    back = hc.check_structure(framed, parts)
    assert back > 0                                     # linked blocks: some match reaches into the previous block
    rc, out = o.orc_decode(o.CODEC_LZ4, framed, src.size)
    assert rc == 0 and np.array_equal(out, src)
    if o.have_ref():
        for T in (1, 3):
            rc, out, _ = o.ref_decompress(o.CODEC_LZ4, framed, src.size, threads=T)
            assert rc == 0 and np.array_equal(out, src)


def test_text_matches_reach_into_the_previous_block():
    src = z.gen_stream(z.GEN_TEXT, 4 * hc.BLOCK, 1 << 20)
    framed = hc.twin_compress(src, 1 << 20, 10)
    assert hc.check_structure(framed, [src]) > 0


def test_ratio_rises_with_the_level_on_text():
    src = z.gen_stream(z.GEN_TEXT, 1 << 20, 1 << 20)
    sizes = [hc.twin_compress(src, 1 << 20, lv).size for lv in hc.LEVELS]
    assert sizes[0] >= sizes[1] >= sizes[2]
    assert sizes[0] < o.orc_encode_lz4(src).size        # level 10 beats the level-1 class


LEVEL_PROBE = r"""
import ctypes, os, sys
L = ctypes.CDLL(sys.argv[1]); L.LZ4MT_createCCtx.restype = ctypes.c_void_p; L.LZ4MT_freeCCtx.argtypes = [ctypes.c_void_p]
for lv in [int(x) for x in sys.argv[2:]]:
    c = L.LZ4MT_createCCtx(2, lv, 1 << 20)
    print(lv, 1 if c else 0, flush=True)
    if c: L.LZ4MT_freeCCtx(c)
"""


def probe(levels, strict):
    env = dict(os.environ)
    env.pop("ZSTDMT_B200_QUIET", None)
    env.pop("ZSTDMT_B200_STRICT_LEVEL", None)
    if strict:
        env["ZSTDMT_B200_STRICT_LEVEL"] = "1"
    r = subprocess.run([sys.executable, "-c", LEVEL_PROBE, z.LIB_PATH] + [str(x) for x in levels], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    ok = {int(a): int(b) for a, b in (line.split() for line in r.stdout.split("\n") if line.strip())}
    said = [line for line in r.stderr.split("\n") if line.strip()]
    return ok, said


@pytest.mark.parametrize("first", [3, 9])
def test_lz4_level_notices_and_strict_table(first):
    """Levels 1-2 and 10-12 are implemented; 3-9 run the level-2 class with a notice (once per process) and are refused
    under ZSTDMT_B200_STRICT_LEVEL=1."""
    ok, said = probe([10, 11, 12], strict=False)
    assert ok == {10: 1, 11: 1, 12: 1} and not said
    others = [lv for lv in range(3, 10) if lv != first]
    ok, said = probe([12, first] + others + [10], strict=False)
    assert all(ok.values()) and len(said) == 1
    assert "lz4 level %d" % first in said[0] and "level-2 search class" in said[0]
    ok, said = probe(list(range(1, 13)), strict=True)
    assert ok == {lv: int(lv <= 2 or lv >= 10) for lv in range(1, 13)} and not said
