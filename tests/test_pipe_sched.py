"""The GPU schedule of the LZ4 level-1 compressor (and of the zstd level-3 encoder on the same front end), restated by
tests/_pipesched.py, gives the CPU twin's candidate offsets and blocks byte for byte, on the edge corpus of
tests/_pipecorpus.py and on generic inputs; every corpus case reaches the edges it is built for and fails its
predicate without its constructions; the invariants the kernel relies on hold on every tile; and two wrong schedule
rules are each caught by a named case.  No GPU involved."""
import os
import re
from collections import defaultdict

import numpy as np
import pytest

import _oracle as o
import _pipecorpus as pc
import _pipesched as ps
import _searchcorpus as sc
import zstdmt_b200 as z

EVENTS = ["period_beats_table", "collision_verify_fails", "first_quad_d_gt_k", "repeat_in_round_no_candidate",
          "insert_skipped_same_hash", "insert_stands_later_past_mflimit",
          "entry_min", "entry_in_match_seg0", "entry_in_match_seg1",
          "w1_merge_v_bit", "w1_merge_free_start", "w1_merge_same_match", "w1_boundary_other_offset",
          "w1_leave_free", "w1_leave_in_match", "w1_last_segment_exhausted", "w1_segment_exhausted",
          "nibble15_shared_by_walk1", "inwarp_path_steps", "path_warps", "warp_without_path_chain", "link_skips_warp",
          "cont_len", "match_ends_on_boundary", "cont_offset_from_pending", "segprev_from_earlier_warp",
          "fold_same_offset", "fold_after_cont", "first_piece_extends_pending", "tile_without_head",
          "tile_skipped_while_pending", "pieces", "ppt", "spt", "nlong", "flush_long_literals_and_long_match",
          "pending_long_literals_from_earlier_tile", "csize_minus_n", "block_shorter_than_16"]


def model_vs_twin(parts, mutant=None):
    """Runs the model on every chunk; asserts its offsets and blocks equal the twin's.  Returns (events, twin
    sequences per chunk and block)."""
    ev, seqs = defaultdict(list), []
    for c, part in enumerate(parts):
        out, _ = ps.lz4_chunk(part, ev, mutant)
        row = []
        for b, (blk, s, off) in enumerate(out):
            src = part[b * ps.BLK: (b + 1) * ps.BLK]
            assert np.array_equal(off, o.lz4_b200_offsets(src).astype(np.int64)), ("offsets differ", c, b)
            tw = o.lz4_block_b200(src)
            if tw.size >= src.size:
                assert blk is None, ("the model writes a block the twin stores", c, b)
            else:
                assert blk is not None and blk == tw.tobytes(), ("the model's block differs from the twin's", c, b)
            assert s == ps.parse_block(tw.tobytes()), ("the model's sequences differ from the twin's", c, b)
            row.append(s)
        seqs.append(row)
    return ev, seqs


BUILT = {b.__name__: b() for b in pc.BUILDERS}
EV = {}


def case_events(name):
    if name not in EV:
        src, chunk, marks, check = BUILT[name]
        EV[name] = model_vs_twin(pc.parts(src, chunk, marks)) + (marks, check)
    return EV[name]


@pytest.mark.parametrize("name", list(BUILT))
def test_corpus_case_reaches_its_edges(name):
    ev, seqs, marks, check = case_events(name)
    check(ev, seqs, marks)


@pytest.mark.parametrize("name", list(BUILT))
def test_predicate_fails_without_the_construction(name):
    src, chunk, marks, check = getattr(pc, name)(knock_out=True)
    ev, seqs = model_vs_twin(pc.parts(src, chunk, marks))
    with pytest.raises(AssertionError):
        check(ev, seqs, marks)


def all_events():
    ev = defaultdict(list)
    for name in BUILT:
        for k, v in case_events(name)[0].items():
            ev[k] += v
    return ev


def test_every_named_event_is_reached(capsys):
    ev = all_events()
    assert set(EVENTS) <= {k for k, v in ev.items() if v}, set(EVENTS) - {k for k, v in ev.items() if v}
    # Density.  Let d_j say that a match is still open at the start of segment j (a Cont piece or E = 0 there).
    # Segment j holds at most 4 + d_j - d_{j+1} piece starts: after a Cont piece of E >= 1 bytes there is room for 4
    # non-Cont starts (E, E + 4, E + 8, E + 12; the last one spills into the next segment, so the match is not open at
    # s_{j+1}), or for 3 when the last one ends on s_{j+1}.  A segment entered free at offset f >= 1 holds 4 starts, or
    # 3 if it closes a match on its end boundary.  The one exception is a segment entered free at offset 0 that closes
    # on its end boundary (starts 0, 4, 8, 12), +1 over the bound.  Inside a tile that state follows a segment at least
    # 1 below the bound (a spill ending exactly on s_j leaves segment j - 1 empty; a free gap before s_j leaves room
    # for one start less).  So
    # only the tile's entry adds one: either free at offset 0 or inside a match (d_{k0} = 1).  The sum telescopes to
    # np <= 4 * 256 + 1 = 1025 (the model asserts it on every tile).  So ppt reaches 5 < C_MAXPIECE / P_TEAM only with
    # 1025 pieces, and densest_tile builds exactly that.  Non-Cont pieces number <= 1024 (hidx) and a tile closes <=
    # 1024 sequences (nemit <= LZ_SPT * P_TEAM, spt <= 4).  A long-literal job needs > 32 literals and a 4-byte match:
    # <= 4096 / 37 + 2 per tile, inside LzBack::longl.
    assert max(ev["ppt"]) == 5 and max(ev["pieces"]) == 4 * ps.C_CHAINS + 1 <= ps.C_MAXPIECE
    assert max(ev["spt"]) == 4
    assert 100 <= max(ev["nlong"]) <= ps.LONGL_WORDS // 2
    # The parse leaves a tile at most one segment past its end (a piece starts before t1 and is cut at t1 + 16 at
    # the latest), so the next tile's entry is in its segment 0 or 1: k0 <= 1, and the "parse already passed this
    # tile" branch of lz_chains (e >= t1) is unreachable; the model records it if it ever runs.
    assert set(ev["k0"]) == {0, 1} and not ev.get("parse_passed_tile")
    assert set(ev["entry_form"]) >= {"walk0_start", "v_bit"}
    assert max(ev["warp_hops"]) <= 8 and max(ev["inwarp_path_steps"]) == 31
    with capsys.disabled():
        print("\n[pipe] max pieces %d, ppt %d, spt %d, nlong per tile %d (longl holds %d), warp hops %d, k0 %s" % (
            max(ev["pieces"]), max(ev["ppt"]), max(ev["spt"]), max(ev["nlong"]), ps.LONGL_WORDS // 2, max(ev["warp_hops"]),
            sorted(set(ev["k0"]))))


# each mutant of the schedule and the corpus case that catches it (its output differs from the twin's, or it trips an
# invariant of the model)
MUTANT_CASES = {"own_from_segment_start": "walks", "head_prev_piece_offset": "marking"}


@pytest.mark.parametrize("mutant", ps.MUTANTS)
def test_schedule_mutant_is_caught(mutant):
    src, chunk, marks, _ = BUILT[MUTANT_CASES[mutant]]
    with pytest.raises(AssertionError):
        model_vs_twin(pc.parts(src, chunk, marks), mutant)


def _struct_array(src, struct, field):
    body = re.search(r"struct[^{]*\b%s\b\s*\{(.*?)\n\};" % struct, src, re.S).group(1)
    return re.search(r"\b%s\[(.+?)\];" % field, body).group(1)


def test_model_constants_match_the_kernels():
    """The model's constants are the #defines of lz4_kernels.cu / lz4_pipe.cuh, and its long-job capacity the size
    of LzBack::longl."""
    k = lambda name: sc.kernel_constant(name, ("lz4_kernels.cu", "lz4_pipe.cuh"))
    assert (ps.C_TILE, ps.C_SEG, ps.C_ROUND, ps.C_HASHLOG) == (k("C_TILE"), k("C_SEG"), k("C_ROUND"), k("C_HASHLOG"))
    assert (ps.C_MAXPIECE, ps.C_LONGLIT, ps.LZ_SPT, ps.P_TEAM) == (k("C_MAXPIECE"), k("C_LONGLIT"), k("LZ_SPT"), k("P_TEAM"))
    assert (ps.C_CHAINS, ps.BLK) == (k("C_CHAINS"), k("LZ4_BLK"))
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zstdmt_b200", "csrc")
    expr = _struct_array(open(os.path.join(csrc, "lz4_kernels.cu")).read(), "LzBack", "longl")
    expr = re.sub(r"\b([A-Z_][A-Z0-9_]*)\b", lambda m: str(k(m.group(1))), expr).replace("/", "//")
    assert ps.LONGL_WORDS == eval(expr)


def kinds():
    rng = np.random.default_rng(78)
    per = lambda p, n: np.resize(rng.integers(0, 256, p, dtype=np.uint8), n)
    yield "text", z.gen_stream(z.GEN_TEXT, 140000, 1 << 20)
    yield "mix", z.gen_stream(z.GEN_MIX, 140000, 1 << 20, first=2)
    yield "zeros", np.zeros(70000, np.uint8)
    yield "random", rng.integers(0, 256, 50000, dtype=np.uint8)
    for p in (1, 2, 3, 4):
        yield "period%d" % p, per(p, 30000 + 4097 * p)
    yield "small-alphabet", rng.integers(0, 3, 80000, dtype=np.uint8)
    yield "short", np.array([1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2], np.uint8)


KINDS = dict(kinds())


@pytest.mark.parametrize("kind", list(KINDS))
def test_model_equals_twin_on_kinds(kind):
    model_vs_twin([KINDS[kind][i: i + ps.BLK] for i in range(0, KINDS[kind].size, ps.BLK)])
