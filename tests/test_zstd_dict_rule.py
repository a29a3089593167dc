"""CPU tests of the zstd dictionary rule: the C ABI of the dictionary calls, and the host walk
(zmt_zstd_scan_frame_dict_host) on frames libzstd writes against trained, finalized and raw-content dictionaries.

The walk names ZB_DICT as the describer of a table exactly where a block uses treeless literals or a Repeat_Mode table
before any block of its frame described one; the expectation is computed here from the frames' section headers, read
independently of the library."""
import ctypes
import re

import numpy as np
import pytest

import zstdmt_b200 as z
import _zdict as zd
from test_frame_index_abi import _header

SYMBOLS = ("zmt_zstd_ddict_bytes", "zmt_zstd_ddict_load_device", "zmt_zstd_scan_frame_dict_host", "zmt_zstd_index_dict_device",
           "zmt_zstd_index_plain_dict_device", "zmt_zstd_blocks_dict_device", "zmt_zstd_decompress_dict_device")
ST_UNSUPPORTED, ST_DICT_WRONG = 10, 13

BLK = np.dtype([("comp_off", "<u8"), ("comp_size", "<u4"), ("frame", "<u4"), ("type", "<u4"), ("regen_hint", "<u4"), ("nseq", "<u4"),
                ("first", "<u4"), ("seq_off", "<u8"), ("lit_off", "<u8"), ("huf_src", "<u4"), ("ll_src", "<u4"), ("of_src", "<u4"),
                ("ml_src", "<u4")])


def test_dictionary_symbols_are_declared_and_exported():
    txt, L = _header(), z.lib()
    for s in SYMBOLS:
        assert re.search(r"\b%s\s*\(" % s, txt), "not declared: " + s
        assert hasattr(L, s), "not exported: " + s
    for base in ("index", "index_plain", "blocks", "decompress"):
        assert getattr(L, "zmt_zstd_%s_dict_device" % base).argtypes[:-1] == getattr(L, "zmt_zstd_%s_device" % base).argtypes
    assert re.search(r"#define\s+ZMT_ST_DICT_WRONG\s+13u", txt) and re.search(r"#define\s+ZF_DICT\s+8u", txt)
    assert z.ST_NAMES[ST_DICT_WRONG] == "dict_wrong"


def test_dict_info_layout_matches_the_header():
    body = re.search(r"typedef struct \{([^{}]*)\} zmt_zstd_dict_info;", _header(), flags=re.S).group(1)
    fields = re.findall(r"(uint32_t|uint64_t)\s+(\w+);", body)
    assert [n for _, n in fields] == [n for n, _ in z.DictInfo._fields_]
    for (t, n), (_, ct) in zip(fields, z.DictInfo._fields_):
        assert ctypes.sizeof(ct) == (4 if t == "uint32_t" else 8), n
    assert ctypes.sizeof(z.DictInfo) == 32
    assert z.lib().zmt_zstd_ddict_bytes() >= ctypes.sizeof(z.DictInfo)


def info_of(d):
    """The summary the device load writes, from the dictionary's first bytes (the walk reads status, ID and kind only)."""
    i = z.DictInfo()
    formatted = zd.dict_id(d) != 0 or (len(d) >= 8 and int(np.asarray(d[:4], np.uint8).view("<u4")[0]) == zd.DICT_MAGIC)
    i.status, i.dict_id, i.kind = 0, zd.dict_id(d), 1 if formatted else 0
    return i


def scan(frame, info):
    """zmt_zstd_scan_frame_dict_host on one frame: (status, flags, descriptors)."""
    L = z.lib()
    frame = np.ascontiguousarray(frame, np.uint8)
    assert L.zmt_zstd_blk_desc_bytes() == BLK.itemsize
    cap = frame.size // 3 + 4
    out = np.zeros(cap, BLK)
    nb, scr, cs, fl = z.c_u32(0), z.c_u64(0), z.c_u64(0), z.c_u32(0)
    args = (frame.ctypes.data, frame.size, 0, 0, out.ctypes.data, ctypes.byref(nb), cap, ctypes.byref(scr), ctypes.byref(cs), ctypes.byref(fl))
    rc = L.zmt_zstd_scan_frame_dict_host(*args, ctypes.byref(info) if info is not None else None)
    return rc, fl.value, out[: nb.value]


def expected_sources(frame, dictionary):
    """Per block (huf_src is ZB_DICT, [ll, of, ml]_src is ZB_DICT), read from the section headers: a treeless section or a
    Repeat_Mode table before any describer of that table in the frame takes the dictionary's (formatted dictionaries only)."""
    f = np.asarray(frame, np.uint8)
    fhd = int(f[4]); single, did, fcs = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    pos = 5 + (0 if single else 1) + [0, 1, 2, 4][did] + [1 if single else 0, 2, 4, 8][fcs]
    described = [False] * 4
    out = []
    while True:
        bh = int(f[pos]) | int(f[pos + 1]) << 8 | int(f[pos + 2]) << 16; pos += 3
        last, typ, bs = bh & 1, (bh >> 1) & 3, bh >> 3
        if typ == 2:
            s = f[pos: pos + bs]
            b0 = int(s[0]); lt, sf = b0 & 3, (b0 >> 2) & 3
            if lt < 2:
                lhdr = 1 if sf in (0, 2) else 2 if sf == 1 else 3
                lregen = (b0 >> 3) if lhdr == 1 else (b0 >> 4) | int(s[1]) << 4 | ((int(s[2]) << 12) if lhdr == 3 else 0)
                lcomp = lregen if lt == 0 else 1
            else:
                lhdr = 3 if sf < 2 else 4 if sf == 2 else 5
                v = int.from_bytes(bytes(s[:lhdr]), "little")
                lcomp = (v >> 14) & 0x3FF if lhdr == 3 else (v >> 18) & 0x3FFF if lhdr == 4 else (v >> 22) & 0x3FFFF
            q = s[lhdr + lcomp:]
            q0 = int(q[0]); used = 1 if q0 < 128 else 2 if q0 < 255 else 3
            nseq = 0 if q0 == 0 else q0 if q0 < 128 else ((q0 - 128) << 8) + int(q[1]) if q0 < 255 else int(q[1]) + (int(q[2]) << 8) + 0x7F00
            huf = lt == 3 and not described[0]
            if lt == 2:
                described[0] = True
            seq = [False] * 3
            if nseq:
                modes = int(q[used])
                for t in range(3):
                    m = (modes >> (6 - 2 * t)) & 3
                    if m == 3:
                        seq[t] = not described[t + 1]
                    else:
                        described[t + 1] = True
            out.append((huf and dictionary, [x and dictionary for x in seq]))
        else:
            out.append((False, [False] * 3))
        pos += bs if typ != 1 else 1
        if last:
            return out


def corpus():
    """(name, dictionary, frames): trained and finalized dictionaries at several levels, and raw content."""
    recs = zd.records(11, 60)
    rng = np.random.default_rng(5)
    cases = []
    for name, d in (("trained_16k", zd.train(1, 16 << 10)), ("trained_112k", zd.train(2, 112 << 10)),
                    ("finalized_32k", zd.finalize(3, np.concatenate(zd.records(9, 40))[: 24 << 10], 32 << 10, dict_id=0x1234567)),
                    ("raw_8k", np.concatenate(zd.records(4, 20))[: 8 << 10])):
        kind = zd.DCT_RAW if name.startswith("raw") else zd.DCT_AUTO
        frames = []
        for lvl in (1, 3, 9, 19):
            for r in recs[lvl % 7:: 9][:4]:
                frames.append(zd.compress(r, d, level=lvl, checksum=int(rng.integers(0, 2)), content_size=int(rng.integers(0, 2)), kind=kind))
        cases.append((name, d, frames))
    return cases


@pytest.fixture(scope="module")
def cases():
    return corpus()


def test_walk_names_the_dictionary_exactly_where_a_first_table_is_reused(cases):
    seen = {"huf": 0, "ll": 0, "of": 0, "ml": 0}
    for name, d, frames in cases:
        info = info_of(d)
        for i, fr in enumerate(frames):
            rc, fl, blk = scan(fr, info)
            assert rc == 0, (name, i, rc)
            assert fl & (zd.ZF_DICT | zd.ZF_NEEDS_SEQ) == zd.ZF_DICT | zd.ZF_NEEDS_SEQ, (name, i)
            exp = expected_sources(fr, info.kind == 1)
            assert len(exp) == blk.size, (name, i)
            for b, (huf, seq) in zip(blk, exp):
                assert (int(b["huf_src"]) == zd.ZB_DICT) == huf, (name, i)
                for t, k in enumerate(("ll_src", "of_src", "ml_src")):
                    assert (int(b[k]) == zd.ZB_DICT) == seq[t], (name, i, k)
                seen["huf"] += huf
                for t, k in enumerate(("ll", "of", "ml")):
                    seen[k] += seq[t]
            if info.kind == 0:
                assert not np.isin(blk[["huf_src", "ll_src", "of_src", "ml_src"]].view("<u4"), [zd.ZB_DICT]).any(), (name, i)
    # libzstd reuses the dictionary's tables in block 0 somewhere in the corpus: every table kind is exercised
    assert all(v > 0 for v in seen.values()), seen


def test_a_frame_naming_another_id_is_dict_wrong(cases):
    name, d, frames = next(c for c in cases if c[0] == "finalized_32k")
    info = info_of(d)
    fr = next(f for f in frames if int(f[4]) & 3)
    assert scan(fr, info)[0] == 0
    info.dict_id ^= 1
    assert scan(fr, info)[0] == ST_DICT_WRONG
    raw = info_of(np.zeros(100, np.uint8))                 # raw content has ID 0: a frame naming one is also DICT_WRONG
    assert raw.kind == 0 and scan(fr, raw)[0] == ST_DICT_WRONG


def test_without_a_dictionary_the_walk_is_unchanged(cases):
    for name, d, frames in cases:
        for fr in frames:
            rc, fl, blk = scan(fr, None)
            if int(fr[4]) & 3:
                assert rc == ST_UNSUPPORTED, name                # a frame naming an ID: refused as before
            else:
                assert rc == 0 and not fl & zd.ZF_DICT, name     # without an ID the walk cannot know; no ZB_DICT is named
                assert not np.isin(blk[["huf_src", "ll_src", "of_src", "ml_src"]].view("<u4"), [zd.ZB_DICT]).any()
    name, d, frames = next(c for c in cases if c[0] == "finalized_32k")
    fr = zd.compress(zd.records(11, 1)[0], d, dict_id_flag=0)
    assert not int(fr[4]) & 3
    rc, fl, _ = scan(fr, info_of(d))
    assert rc == 0 and fl & zd.ZF_DICT                         # a frame naming no ID takes the batch's dictionary


def test_a_failed_load_fails_every_frame(cases):
    name, d, frames = cases[0]
    info = info_of(d)
    info.status = 3
    assert all(scan(fr, info)[0] == 3 for fr in frames)
