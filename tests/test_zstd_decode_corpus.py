"""CPU tests of the zstd edge corpus (_zcorpus.py): every frame decodes to its source in libzstd and in the oracle, every
case reaches the edge it exists for, and the host scan of the GPU decoder (zmt_zstd_scan_frame_host) describes each
frame as the oracle's block trace does."""
import ctypes

import numpy as np
import pytest

import _oracle as o
import _zcorpus as zc
import zstdmt_b200 as z

ZT = zc.ZT
CASES = list(zc.CASES)

# ZBlk of zstd_decode.cu
ZBLK = np.dtype([("comp_off", "<u8"), ("comp_size", "<u4"), ("frame", "<u4"), ("type", "<u4"), ("regen_hint", "<u4"),
                 ("nseq", "<u4"), ("first", "<u4"), ("seq_off", "<u8"), ("lit_off", "<u8"),
                 ("huf_src", "<u4"), ("ll_src", "<u4"), ("of_src", "<u4"), ("ml_src", "<u4")])
SELF, PREDEF, NONE = 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD
ZF_NEEDS_SEQ, ZF_CHECKSUM, ZF_NO_SIZE = 1, 2, 4


def host_scan(frame, frame_idx=0, first_block=0):
    """zmt_zstd_scan_frame_host on one frame: (status, block descriptors, content size, frame flags)."""
    L = z.lib()
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    cap = frame.size // 3 + 16
    buf = np.zeros(cap * ZBLK.itemsize, np.uint8)
    nblk, scr, cs, flags = ctypes.c_uint32(first_block), ctypes.c_uint64(0), ctypes.c_uint64(0), ctypes.c_uint32(0)
    out = np.zeros((cap + first_block) * ZBLK.itemsize, np.uint8)
    rc = L.zmt_zstd_scan_frame_host(frame.ctypes.data, frame.size, 0, frame_idx, out.ctypes.data, ctypes.byref(nblk), cap + first_block,
                                    ctypes.byref(scr), ctypes.byref(cs), ctypes.byref(flags))
    return rc, out.view(ZBLK)[first_block: nblk.value], cs.value, flags.value


def expected_flags(frame, tr):
    """The frame flags restated from the header and the trace: NEEDS_SEQ exactly when some block has treeless literals or a
    sequences section with a non-predefined table."""
    fhd = int(frame[4])
    seq = (tr.col("lit_type") == 3).any() or ((tr.col("nseq") > 0) & (tr.col("modes") != 0)).any()
    return (ZF_NEEDS_SEQ if seq else 0) | (ZF_CHECKSUM if fhd & 4 else 0) | (ZF_NO_SIZE if (fhd >> 6) == 0 and not (fhd & 0x20) else 0)


def expected_sources(tr, base):
    """Per block: (huf_src, ll_src, of_src, ml_src) restated from the trace.  Treeless literals take the tree of the last
    block with Huffman literals of its own; a table in Repeat_Mode is the one the last block with mode 1 or 2 for that
    table described, or the predefined one after a mode-0 block.  Blocks that describe their own (or have no sequences)
    are SELF, predefined tables PREDEF.  Indices are batch-wide (base = index of the frame's first block)."""
    lt, m = tr.col("lit_type"), zc.modes(tr)
    rep = {(r["block"], r["table"]): r["src"] for r in zc.repeat_sources(tr)}
    last_huf, out = NONE, []
    for b in range(len(lt)):
        huf = SELF
        if lt[b] == 2:
            last_huf = base + b
        elif lt[b] == 3:
            huf = last_huf
        t3 = []
        for t in range(3):
            if m[b, t] == 3:
                s = rep[(b, t)]
                t3.append(NONE if s is None else PREDEF if s == "predef" else base + s)
            else:
                t3.append(PREDEF if m[b, t] == 0 else SELF)
        out.append((huf, *t3))
    return out


def test_block_descriptor_is_64_bytes():
    assert z.lib().zmt_zstd_blk_desc_bytes() == 64 == ZBLK.itemsize


def test_libzstd_version_and_parameter_ids():
    """The corpus relies on experimental parameter ids of libzstd 1.5.x; the module checks them through their bounds."""
    L = zc.zstd()
    assert L.ZSTD_versionNumber() // 100 == 105
    for pid, want in zc.EXPECT_BOUNDS.items():
        b = L.ZSTD_cParam_getBounds(pid)
        assert (b.lowerBound, b.upperBound) == want


@pytest.mark.parametrize("name", CASES)
def test_corpus_case_reaches_its_edge(name):
    """Each case's own predicate on the oracle's block trace: the edge it exists for is in the frame libzstd wrote."""
    assert zc.CASES[name][1](zc.trace(name)), name


@pytest.mark.parametrize("name", CASES)
def test_corpus_frame_restores_source_in_libzstd_and_oracle(name):
    """Content and parse agree: libzstd and the oracle's RFC 8878 decoder both restore the source the parse built."""
    src, frame = zc.case(name)
    assert np.array_equal(zc.libzstd_decompress(frame, src.size), src)
    out = np.empty(src.size + 1, np.uint8); got, used = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = o.orc().orc_zstd_decode(frame.ctypes.data, frame.size, out.ctypes.data, out.size, ctypes.byref(got), ctypes.byref(used))
    assert rc == 0 and used.value == frame.size
    assert np.array_equal(out[: got.value], src)
    assert np.array_equal(zc.trace(name).content, src)


@pytest.mark.parametrize("base", [0, 5])
@pytest.mark.parametrize("name", CASES)
def test_host_scan_agrees_with_trace(name, base):
    """zmt_zstd_scan_frame_host against the oracle's trace, block by block: type, sizes, sequence count, the frame flags,
    and the block it names as the source of every inherited Huffman tree and sequence table (which the dependent-block
    kernel rebuilds the tables from).  base: the frame's first block is not block 0 of the batch."""
    src, frame = zc.case(name)
    tr = zc.trace(name)
    rc, blk, cs, flags = host_scan(frame, frame_idx=3, first_block=base)
    assert rc == 0
    assert len(blk) == len(tr.blk)
    assert cs == src.size
    assert flags == expected_flags(frame, tr)
    typ = tr.col("type")
    assert list(blk["type"]) == list(typ)
    assert (blk["frame"] == 3).all() and list(blk["first"]) == [1] + [0] * (len(blk) - 1)
    assert list(blk["regen_hint"]) == [int(r if t != 2 else l) for t, r, l in zip(typ, tr.col("regen"), tr.col("lit_regen"))]
    assert list(blk["comp_size"]) == [int(1 if t == 1 else s) for t, s in zip(typ, tr.col("bsize"))]
    assert list(blk["nseq"]) == [max(0, int(n)) for n in tr.col("nseq")]
    exp = expected_sources(tr, base)
    for b in np.flatnonzero(typ == 2):
        got = tuple(int(blk[k][b]) for k in ("huf_src", "ll_src", "of_src", "ml_src"))
        assert got == exp[b], (name, int(b), [hex(x) for x in got], [hex(x) for x in exp[b]])


def test_host_scan_sources_point_back_further_than_one_block():
    """The restatement above is not vacuous: in `tables` some Repeat_Mode table is described two or more blocks back, and
    in `literals` some treeless block's tree is not the previous block's."""
    tr = zc.trace("tables")
    assert any(r["src"] not in (None, "predef") and r["src"] < r["block"] - 1 for r in zc.repeat_sources(tr))
    ex = expected_sources(zc.trace("literals"), 0)
    assert any(h not in (SELF, NONE) and h < b - 1 for b, (h, *_) in enumerate(ex))
