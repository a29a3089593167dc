"""CPU tests of the models of the zstd execute pass and lane sequence reader (_zxmodel.py) on the whole zstd edge corpus
(_zcorpus.py): each x_* case reaches every edge it names, the execute steps partition every block as zx_block cuts it,
the kernel's dependency search agrees with the pairwise overlap, the lane reader decodes every predefined-table block to
the oracle's sequences and never runs out of bits, the model's constants are the kernel's, and each case's predicate
fails when its edge blocks are left out of the parse."""
import numpy as np
import pytest

import _zcorpus as zc
import _zxmodel as zx
from test_zstd_decode_corpus import host_scan

CASES = list(zc.CASES)
X_CASES = list(zc.X_CASES)


def test_model_constants_match_the_kernel():
    """The model's constants are the ones zstd_decode.cu states; a change in either fails here instead of the model
    quietly following the code."""
    k = zx.kernel_constants()
    assert k == {"ZX_SPAN": zx.ZX_SPAN, "STEP_CAP": zx.STEP_CAP, "LANE_LIT": zx.LANE_LIT, "LANE_LIT_WARP": zx.LANE_LIT,
                 "OWN_ML": zx.OWN_ML, "OWN_ML_BALLOT": zx.OWN_ML, "CHUNK": zx.CHUNK, "REFILL_AT": zx.REFILL_AT,
                 "OFC_MAX": zx.OFC_MAX, "INACTIVE": zx.INACTIVE}


def test_predefined_tables_budget():
    """The lane reader's budget: after a refill at least 57 bits are valid; the three state updates take at most
    6 + 6 + 5 = 17 bits, so REFILL_AT + 17 == 57; offset codes up to OFC_MAX with 16 + 16 extra bits would not fit
    without the second refill."""
    assert max(nb for _, nb, _ in zx.T_LL) + max(nb for _, nb, _ in zx.T_ML) + max(nb for _, nb, _ in zx.T_OF) == 17
    assert zx.REFILL_AT + 17 == 57
    for t, log in ((zx.T_LL, 6), (zx.T_ML, 6), (zx.T_OF, 5)):
        assert len(t) == 1 << log and all(0 <= base + (1 << nb) - 1 < (1 << log) for _, nb, base in t)
    assert [zx.LL_BASE[c + 1] - zx.LL_BASE[c] for c in range(35)] == [1 << b for b in zx.LL_BITS[:35]]
    assert [zx.ML_BASE[c + 1] - zx.ML_BASE[c] for c in range(52)] == [1 << b for b in zx.ML_BITS[:52]]


def check_steps(tr, b, r):
    """The steps of one block: in order, each prefix-maximal under the sequence cap and the span, lone exactly when the
    first sequence alone exceeds the span; their bytes plus the trailing literals are the block's regenerated size."""
    q = tr.block_seqs(b).astype(np.int64)
    sizes = q[:, 0] + q[:, 2]
    nxt, op, lp = 0, 0, 0
    for s in r["steps"]:
        assert s["first"] == nxt and (s["op"], s["lp"]) == (op, lp)
        a, n = s["first"], s["n"]
        assert s["span"] == int(sizes[a: a + n].sum())
        if s["kind"] == "lone":
            assert n == 1 and sizes[a] > zx.ZX_SPAN
        else:
            assert n <= zx.STEP_CAP and s["span"] <= zx.ZX_SPAN
            more = a + n < len(q)
            assert not more or n == zx.STEP_CAP or s["span"] + sizes[a + n] > zx.ZX_SPAN, "a step stops short"
            assert s["end"] == ("end" if not more else "cap" if n == zx.STEP_CAP else "span")
        nxt += n; op += s["span"]; lp += int(q[a: a + n, 0].sum())
    assert nxt == len(q)
    assert op + r["trailing"] == tr.col("regen")[b] and lp + r["trailing"] == tr.col("lit_regen")[b]


@pytest.mark.parametrize("name", CASES)
def test_execute_model_on_every_case(name):
    """Every compressed block of every case: the steps partition its sequences as zx_block cuts them, and the kernel's
    dependency search (lower bound over lanes) gives the pairwise overlap's answer on every record."""
    tr = zc.trace(name)
    blocks, _ = zx.exec_frame(tr)
    assert blocks or not (tr.col("nseq") > 0).any()
    for b, r in blocks.items():
        check_steps(tr, b, r)
        assert all(s["dep"] == s["dep_kernel"] for s in r["seqs"] if s["match"] != "lone")
        for s in r["seqs"]:
            if s["match"] == "own":
                assert s["indep"] and s["off"] >= s["ml"] and s["ml"] <= zx.OWN_ML and 0 <= s["nlow"] <= s["ml"]


def test_dependency_search_equals_overlap_on_constructed_lanes():
    """The two formulations on every source start around every destination edge of a step of three matches, with the
    inactive lanes the kernel pads with."""
    mp, ml = [10, 30, 31], [5, 1, 20]
    d_beg = mp + [zx.INACTIVE] * 29
    e_end = [m + n for m, n in zip(mp, ml)] + [zx.INACTIVE] * 29
    for lane in range(1, 3):
        for sp in range(0, mp[lane]):
            for n in (1, 3, 8):
                pair = any(mp[j] < sp + n and sp < mp[j] + ml[j] for j in range(lane))
                assert zx.kernel_dependent(lane, sp, n, d_beg, e_end) == pair, (lane, sp, n)


@pytest.mark.parametrize("name", X_CASES)
def test_x_case_reaches_every_event_it_names(name):
    """The events each x_* case names, listed when missing (the case predicate asserts the same, without the list)."""
    tr = zc.trace(name)
    if name == "x_budget":
        lanes, ev = zx.lane_frame(tr.frame)
        want = zc.BUDGET_EVENTS
        assert min(s["slack"] for r in lanes.values() for s in r["seqs"]) == 0
    else:
        ev = zx.exec_frame(tr)[1]
        want = zc.X_EVENTS[name.rsplit("_", 1)[0]]
    assert [e for e in want if not ev[e]] == []
    assert (zc.lane_route if name.endswith(("_l1", "budget")) else zc.dep_route)(tr)


@pytest.mark.parametrize("name", CASES)
def test_lane_reader_decodes_and_never_runs_short(name):
    """Every block the lane decoder takes: the model decodes the oracle's sequences from the block's bytes, consumes the
    bit stream exactly, and leaves no sequence with fewer bits than it reads (slack >= 0)."""
    tr = zc.trace(name)
    lanes, _ = zx.lane_frame(tr.frame)
    for b, r in lanes.items():
        rows = tr.block_seqs(b)[:, :3].astype(np.int64)
        got = np.array([(s["ll"], s["ofv"], s["ml"]) for s in r["seqs"]], np.int64)
        assert np.array_equal(got, rows), (name, b)
        assert min(s["slack"] for s in r["seqs"]) >= 0, (name, b)
        for s in r["seqs"]:
            assert 57 <= s["V"] <= 64 and s["refill2"] == (s["S1"] > zx.REFILL_AT and s is not r["seqs"][-1])
    if name in ("far_predef", "reps_predef", "x_budget") or name.endswith("_l1"):
        assert lanes, name


def test_lane_reader_leaves_the_general_path_its_blocks():
    """None for the blocks the lane kernel hands on: offset codes above 24 (far_predef), a repeat Offset_Value
    (reps_predef), and every block of a frame the host scan flags (tables)."""
    tr = zc.trace("far_predef")
    lanes, _ = zx.lane_frame(tr.frame)
    big = {int(b) for b in np.flatnonzero(tr.col("nseq") > 0) if (zc.of_codes(tr)[zc.seq_blocks(tr) == b] > 24).any()}
    assert big and not big & set(lanes)
    tr = zc.trace("reps_predef")
    lanes, _ = zx.lane_frame(tr.frame)
    rep = {int(b) for b in np.flatnonzero(tr.col("nseq") > 0) if (tr.block_seqs(int(b))[:, 1] <= 3).any()}
    assert rep and not rep & set(lanes)
    assert zx.lane_frame(zc.trace("tables").frame)[0] == {}


@pytest.mark.parametrize("name", ["x_budget", "x_cross_l1", "literals", "reps"])
def test_frame_walk_agrees_with_host_scan(name):
    """The model's frame walk finds every block where zmt_zstd_scan_frame_host does."""
    frame = zc.case(name)[1]
    rc, blk, _, flags = host_scan(frame)
    assert rc == 0
    walk, needs = zx.frame_blocks(frame)
    assert [(t, o) for t, o, _ in walk] == [(int(t), int(o)) for t, o in zip(blk["type"], blk["comp_off"])]
    assert needs == bool(flags & 1)


OMIT = {"x_steps": "lone_off_1", "x_lits": "runs", "x_matches": "chain", "x_cross": "lone_back3"}


@pytest.mark.parametrize("name", X_CASES)
def test_predicate_fails_without_its_edge(name, monkeypatch):
    """The predicates are not vacuous: with one of a case's edge blocks left out of the parse (written as pad), the
    frame still decodes in the oracle, and the predicate fails."""
    label = "s1_55" if name == "x_budget" else OMIT[name.rsplit("_", 1)[0]]
    monkeypatch.setattr(zc.Plan, "omit", frozenset([label]))
    src, seqs, params = zc.CASES[name][0]()
    frame = zc.compress(src, params, seqs)
    tr = zc.o.zstd_trace(frame)
    tr.frame = frame
    assert np.array_equal(tr.content, src)
    assert not zc.CASES[name][1](tr)
