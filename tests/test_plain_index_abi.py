"""CPU tests of the plain-stream frame index's C ABI: the library exports the two calls include/zstdmt_b200_dev.h declares,
their argument lists are those of the container calls, and they report under the existing profiling id."""
import re

import zstdmt_b200 as z
from test_frame_index_abi import _header

PAIRS = (("zmt_lz4_index_plain_device", "zmt_lz4_index_device"), ("zmt_zstd_index_plain_device", "zmt_zstd_index_device"))


def _params(txt, name):
    m = re.search(r"\bint\s+%s\s*\((.*?)\);" % name, txt, flags=re.S)
    assert m, "not declared: " + name
    return [re.sub(r"\s+", " ", p).strip().rsplit(" ", 1)[0] for p in m.group(1).split(",")]


def test_plain_index_symbols_are_declared_and_exported():
    txt, L = _header(), z.lib()
    for plain, container in PAIRS:
        assert _params(txt, plain) == _params(txt, container), plain
        assert hasattr(L, plain), "not exported: " + plain
        assert getattr(L, plain).argtypes == getattr(L, container).argtypes


def test_profiling_id_is_unchanged():
    ids = re.search(r"enum \{(.*?)\};", _header(), flags=re.S).group(1)
    names = [re.sub(r"\s*=.*", "", x).strip() for x in ids.split(",")]
    assert names.index("ZMT_K_FRAME_INDEX") == 16 and names[-1] == "ZMT_K_COUNT" and len(names) == 18


def test_header_states_the_layout_convention_and_every_plain_status():
    txt = open(z.os.path.join(z.os.path.dirname(z._HERE), "include", "zstdmt_b200_dev.h")).read()
    sec = txt[txt.index("Frame index on the device for plain streams"): txt.index("zmt_lz4_index_plain_device(")]
    assert "d_in - 12" in sec and "in_bytes + 12" in sec
    for st in ("TRUNCATED", "BAD_MAGIC", "BAD_HEADER", "CONTENT_SIZE", "UNSUPPORTED", "DST_SMALL", "TRAILING"):
        assert "ZMT_ST_" + st in sec, st
