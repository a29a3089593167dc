"""The CPU twin of the zstd level 6-12 search class (oracle/zstd_lazy_twin.c) against the rule restated in Python
(tests/_zlazy.py), and the level table of ZSTDCB_createCCtx.  No GPU involved."""
import os
import subprocess
import sys

import numpy as np
import pytest

import _zlazy as zl
import zstdmt_b200 as z

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def inputs():
    rng = np.random.default_rng(2024)
    per = lambda p, n: np.resize(rng.integers(0, 256, p, dtype=np.uint8), n)
    yield "text", z.gen_stream(z.GEN_TEXT, 100 << 10, 1 << 20)
    yield "mix", z.gen_stream(z.GEN_MIX, 60000, 1 << 20, first=2)
    yield "zeros", np.zeros(20000, np.uint8)
    yield "random", rng.integers(0, 256, 30000, dtype=np.uint8)
    for p in (1, 2, 3, 4):
        yield "period%d" % p, per(p, 9000 + p)
    yield "small-alphabet", rng.integers(0, 3, 25000, dtype=np.uint8)
    yield "empty", np.zeros(0, np.uint8)
    yield "one", np.array([9], np.uint8)
    yield "short", np.array([1, 2, 3], np.uint8)


CASES = [(name, lv, W, B) for name, _ in inputs() for lv in (6, 9, 12) for W, B in ((0, 0), (4096, 1024), (700, 3000))]
DATA = dict(inputs())


@pytest.mark.parametrize("name,level,W,B", CASES)
def test_twin_equals_restatement_and_replays(name, level, W, B):
    src = DATA[name]
    if level == 12 and name == "text" and not W:
        src = src[: 40 << 10]                          # the restatement walks 64 candidates per position in Python
    want = zl.sequences(src, level, W=W or None, block=B or zl.BLOCK)
    got = zl.twin_sequences(src, level, W, B)
    assert len(got) == len(want)
    for b, (g, w) in enumerate(zip(got, want)):
        assert [tuple(x) for x in g.tolist()] == w, (name, level, W, B, b)
    assert zl.replay(src, want, B or zl.BLOCK) == src.tobytes()
    if W:
        assert all(off <= W for seqs in want for _, off, _ in seqs)


def test_levels_above_12_use_level_12():
    src = DATA["text"][: 30 << 10]
    a = zl.twin_sequences(src, 12)
    for lv in (13, 19, 22):
        b = zl.twin_sequences(src, lv)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


NOTICE_PROBE = r"""
import ctypes, os, sys
L = ctypes.CDLL(sys.argv[1]); L.ZSTDCB_createCCtx.restype = ctypes.c_void_p; L.ZSTDCB_freeCCtx.argtypes = [ctypes.c_void_p]
for lv in [int(x) for x in sys.argv[2:]]:
    c = L.ZSTDCB_createCCtx(2, lv, 0)
    print(lv, 1 if c else 0, flush=True)
    if c: L.ZSTDCB_freeCCtx(c)
"""


def probe(levels, strict):
    env = dict(os.environ)
    env.pop("ZSTDMT_B200_QUIET", None)
    env.pop("ZSTDMT_B200_STRICT_LEVEL", None)
    if strict:
        env["ZSTDMT_B200_STRICT_LEVEL"] = "1"
    r = subprocess.run([sys.executable, "-c", NOTICE_PROBE, z.LIB_PATH] + [str(x) for x in levels], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    ok = {int(a): int(b) for a, b in (line.split() for line in r.stdout.split("\n") if line.strip())}
    said = {int(line.split("level ")[1].split()[0]): line for line in r.stderr.split("\n") if line.strip()}
    return ok, said


def test_zstd_level_notices_and_strict_table():
    """Levels 1-3 and 6-12 are implemented; 4-5 run the level-3 class and 13-22 the level-12 class, each class with a
    notice of its own (once per process), and both refused under ZSTDMT_B200_STRICT_LEVEL=1."""
    ok, said = probe([4, 6, 12, 13, 19, 5], strict=False)
    assert all(ok[lv] for lv in (4, 6, 12, 13, 19, 5))
    assert set(said) == {4, 13}
    assert "level-3 search class" in said[4] and "level-12 search class" in said[13]
    ok, said = probe([19, 4, 3, 6, 12, 13], strict=True)
    assert ok == {19: 0, 4: 0, 3: 1, 6: 1, 12: 1, 13: 0} and not said
