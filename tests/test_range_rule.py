"""CPU tests of the range-read rule (tests/_ranges.py) on the golden streams, and of the range-read C ABI.

On every golden stream only the frames the rule selects are decoded (by the oracle, as a container stream of those frames
alone) and the ranges are gathered from them; the result must equal the same slices of the oracle's decode of the whole
stream."""
import ctypes
import os
import re

import numpy as np
import pytest

import _oracle as o
import _ranges as rr
import zstdmt_b200 as z
from test_frame_index_abi import _header

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SYMBOLS = ("zmt_range_workspace_bytes", "zmt_lz4_content_offsets_device", "zmt_zstd_content_offsets_device", "zmt_lz4_range_plan_device",
           "zmt_zstd_range_plan_device", "zmt_lz4_range_read_workspace_bytes", "zmt_zstd_range_read_workspace_bytes",
           "zmt_lz4_range_read_device", "zmt_zstd_range_read_device")


def golden():
    import json
    with open(os.path.join(GOLD, "manifest.json")) as f:
        return json.load(f)["cases"]


def container(frames):
    parts = []
    for f in frames:
        parts += [np.frombuffer((0x184D2A50).to_bytes(4, "little") + (4).to_bytes(4, "little") + int(f.size).to_bytes(4, "little"), np.uint8), f]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


@pytest.mark.parametrize("case", golden(), ids=lambda c: c["file"])
def test_selected_frames_give_the_slices_of_the_full_decode(case):
    codec = case["codec"]
    cid = o.CODEC_LZ4 if codec == "lz4" else o.CODEC_ZSTD
    fb = np.fromfile(os.path.join(GOLD, case["file"]), dtype=np.uint8)
    frames = o.mt_frames(fb)
    st, _, off = rr.content_table(rr.content_sizes(frames, codec), [f.size for f in frames])
    assert st == rr.ST_OK
    rc, full = o.orc_decode(cid, fb, case["n"] + 16)
    assert rc == 0 and full.size == off[-1] == case["n"]
    ranges = rr.ranges_for(off, np.random.default_rng(case["n"]), nrandom=10000, max_len=3 * case["chunk"])
    p = rr.plan(off, ranges, [f.size for f in frames])
    assert p["sel"] == sorted(set(p["sel"])) and p["dst_off"][-1] == sum(n for _, n in ranges)
    contents = {}
    for f in p["sel"]:                                       # each selected frame decoded on its own, once
        rc, c = o.orc_decode(cid, container([frames[f]]), off[f + 1] - off[f] + 16)
        assert rc == 0 and c.size == off[f + 1] - off[f]
        contents[f] = c
    for (s, n), (st, got) in zip(ranges, rr.apply(off, ranges, p, contents)):
        assert st == rr.ST_OK and np.array_equal(got, full[s: s + n]), (s, n)


def test_rule_spans_statuses_and_layout():
    off = [0, 10, 10, 25, 40]                                # frame 1 is empty
    assert rr.span(off, 0, 1) == (0, 0) and rr.span(off, 9, 2) == (0, 2) and rr.span(off, 10, 1) == (2, 2)
    assert rr.span(off, 24, 2) == (2, 3) and rr.span(off, 0, 40) == (0, 3) and rr.span(off, 39, 1) == (3, 3)
    ranges = [(39, 2), (5, (1 << 64) - 3), (40, 0), (12, 3), (9, 3), (12, 3)]
    p = rr.plan(off, ranges, [20, 5, 30, 30])
    assert p["sel"] == [0, 1, 2] and p["scratch_off"] == [0, 10, 10, 25]
    assert p["dst_off"] == [0, 0, 0, 0, 3, 6, 9] and p["packed"] == 48 + 32 + 48
    contents = {0: np.arange(10, dtype=np.uint8), 1: np.zeros(0, np.uint8), 2: np.arange(100, 115, dtype=np.uint8)}
    got = rr.apply(off, ranges, p, contents, {2: rr.ST_BLOCK})
    assert [s for s, _ in got] == [rr.ST_BAD_ARG, rr.ST_BAD_ARG, rr.ST_OK, rr.ST_BLOCK, rr.ST_BLOCK, rr.ST_BLOCK]
    got = rr.apply(off, ranges, p, contents, {1: rr.ST_CONTENT_CHECKSUM})
    assert got[3][0] == rr.ST_OK and np.array_equal(got[3][1], [102, 103, 104]) and got[4][0] == rr.ST_CONTENT_CHECKSUM
    assert rr.content_table([5, None, 3], [9, 9, 9])[:2] == (rr.ST_UNSUPPORTED, 1)
    assert rr.content_table([5, 9 * 32768 + 1], [9, 9])[:2] == (rr.ST_CONTENT_SIZE, 1)


def test_range_symbols_are_declared_and_exported():
    txt, L = _header(), z.lib()
    for s in SYMBOLS:
        assert re.search(r"\b%s\s*\(" % s, txt), "not declared: " + s
        assert hasattr(L, s), "not exported: " + s


def test_plan_struct_matches_the_header():
    body = re.search(r"typedef struct \{([^{}]*)\} zmt_range_plan;", _header(), flags=re.S).group(1)
    fields = re.findall(r"(uint32_t|uint64_t)\s+(\w+);", body)
    ct = {"uint32_t": ctypes.c_uint32, "uint64_t": ctypes.c_uint64}
    assert [(n, ct[t]) for t, n in fields] == list(z.RangePlan._fields_)
    assert ctypes.sizeof(z.RangePlan) == 64


def test_range_read_scopes_report_under_the_frame_index_id():
    """Range reads add no profiling id: every profiling scope in range_read.cu reports under ZMT_K_FRAME_INDEX, whose
    place and doc line say so."""
    ids = re.search(r"enum \{(.*?)\};", _header(), flags=re.S).group(1)
    names = [re.sub(r"\s*=.*", "", x).strip() for x in ids.split(",")]
    assert names.index("ZMT_K_FRAME_INDEX") == 16 and names[-1] == "ZMT_K_COUNT" and "ZMT_K_RANGE" not in names
    doc = open(os.path.join(os.path.dirname(GOLD), "..", "include", "zstdmt_b200_dev.h")).read()
    assert re.search(r"ZMT_K_FRAME_INDEX = one index call[^/]*range reads report here too", doc, flags=re.S)
    src = open(os.path.join(os.path.dirname(GOLD), "..", "zstdmt_b200", "csrc", "range_read.cu")).read()
    assert set(re.findall(r"ZmtProfScope\s+\w+\((ZMT_K_\w+)", src)) == {"ZMT_K_FRAME_INDEX"}


def test_read_workspace_is_that_of_the_selected_frames():
    L = z.lib()
    plan = z.RangePlan(nframes=64, nranges=1, nsel=1, nunits=16, packed_bytes=(1 << 20) + 16, scratch_bytes=1 << 20)
    want = ((plan.packed_bytes + 255) & ~255) + L.zmt_lz4d_workspace_bytes(1, 16, plan.packed_bytes)
    assert L.zmt_lz4_range_read_workspace_bytes(ctypes.byref(plan)) == want
    plan.nunits, plan.dec_scratch = 8, 4096
    want = ((8 * L.zmt_zstd_blk_desc_bytes() + 255) & ~255) + L.zmt_zstdd_workspace_bytes(1, 8, 4096)
    assert L.zmt_zstd_range_read_workspace_bytes(ctypes.byref(plan)) == want
