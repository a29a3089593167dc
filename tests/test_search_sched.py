"""The GPU schedule of the chain-search encoders (zstd levels 6-12, LZ4 levels 10-12), restated from the CPU twins'
best[] by tests/_searchsched.py, gives the twins' sequences block for block, on the edge corpus of
tests/_searchcorpus.py and on generic inputs; every corpus case reaches the edge it is built for.  No GPU involved."""
from collections import defaultdict

import numpy as np
import pytest

import _lz4hc as hc
import _searchcorpus as sc
import _searchsched as ss
import _zlazy as zl
import zstdmt_b200 as z

CASES = sc.cases()
BY_NAME = {c.name: c for c in CASES}
EVENTS = ["range_no_entry", "entry_is_literal", "match_ends_at_range_end", "match_ends_one_before_range_end",
          "match_ends_one_past_range_end", "match_skips_range", "fold_at_entry", "fold_after_range_without_sequence",
          "carry_from_k_ranges", "defer_looks_into_next_range", "defer_looks_into_next_quarter", "quarter_carry_pos",
          "quarter_entry_fold", "quarter_entry_no_fold", "quarter_entry_literal", "open_across_whole_quarter",
          "held_sequences", "long_jobs"]


def model_vs_twin(codec, parts, level):
    """Runs the model on every chunk's twin best[]; asserts its sequences equal the twin's.  Returns (events, twin
    sequences per chunk and block, twin best[] per chunk)."""
    ev, seqs, bests = defaultdict(list), [], []
    for c, part in enumerate(parts):
        if codec == "zstd":
            tw, best = zl.twin_sequences(part, level), zl.twin_best(part, level)
            got, e = ss.zstd_chunk(best, zl.params(level)[2])
        else:
            tw, best = hc.twin_sequences(part, level), hc.twin_best(part, level)
            got, e = ss.lz4_chunk(best, hc.PARAMS[level][1])
        assert len(got) == len(tw), (c, len(got), len(tw))
        for b, (g, t) in enumerate(zip(got, tw)):
            assert g == [tuple(r) for r in t.tolist()], ("the model's sequences differ from the twin's", c, b)
        for k, v in e.items():
            ev[k] += v
        seqs.append(tw)
        bests.append(best)
    return ev, seqs, bests


@pytest.mark.parametrize("name,level", [(c.name, lv) for c in CASES for lv in c.levels])
def test_corpus_case_reaches_its_edge(name, level):
    case = BY_NAME[name]
    case.check(level, *model_vs_twin(case.codec, sc.parts(case), level))


def test_every_named_event_is_reached():
    seen = set()
    for case in CASES:
        ev = model_vs_twin(case.codec, sc.parts(case), case.levels[0])[0]
        seen |= {k for k, v in ev.items() if v}
    assert set(EVENTS) <= seen, set(EVENTS) - seen
    ev = model_vs_twin("zstd", sc.parts(BY_NAME["zstd_phases"]), 6)[0]
    assert max(ev["carry_from_k_ranges"]) >= 3


def test_model_constants_and_capacities_match_the_kernels():
    """The model's range and quarter are the kernels' ZL_RANGE and L4H_Q, its long-job threshold is their C_LONGLIT,
    and the dense case's bounds fit L4H_MAXSEQ and L4H_MAXLONG as lz4_hc.cuh defines them."""
    assert (ss.RANGE, ss.QUARTER) == (sc.kernel_constant("ZL_RANGE", ("zstd_lazy.cuh",)), sc.kernel_constant("L4H_Q"))
    assert ss.LONGLIT == sc.kernel_constant("C_LONGLIT")
    assert (sc.MAXSEQ, sc.MAXLONG) == (ss.QUARTER // 4 + 2, ss.QUARTER // 33 + ss.QUARTER // 1290 + 8)


def kinds():
    rng = np.random.default_rng(77)
    per = lambda p, n: np.resize(rng.integers(0, 256, p, dtype=np.uint8), n)
    yield "text", z.gen_stream(z.GEN_TEXT, 200 << 10, 1 << 20)
    yield "mix", z.gen_stream(z.GEN_MIX, 200000, 1 << 20, first=2)
    yield "zeros", np.zeros(70000, np.uint8)
    yield "random", rng.integers(0, 256, 50000, dtype=np.uint8)
    for p in (1, 2, 3, 4):
        yield "period%d" % p, per(p, 70000 + p)
    yield "small-alphabet", rng.integers(0, 3, 80000, dtype=np.uint8)
    yield "short", np.array([1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2], np.uint8)


KINDS = dict(kinds())


@pytest.mark.parametrize("codec,level", [("zstd", 6), ("zstd", 8), ("zstd", 12), ("lz4", 10), ("lz4", 12)])
@pytest.mark.parametrize("kind", list(KINDS))
def test_model_equals_twin_on_kinds(kind, codec, level):
    model_vs_twin(codec, [KINDS[kind]], level)
