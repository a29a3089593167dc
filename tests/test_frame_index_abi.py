"""CPU tests of the device frame index's C ABI: the library exports what include/zstdmt_b200_dev.h declares for it, and the
summary struct and profiling id the header defines are the ones the Python binding reads."""
import ctypes
import os
import re

import zstdmt_b200 as z

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "zstdmt_b200_dev.h")
SYMBOLS = ("zmt_index_workspace_bytes", "zmt_lz4_index_device", "zmt_zstd_index_device", "zmt_zstd_blocks_device")


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_index_symbols_are_declared_and_exported():
    txt, L = _header(), z.lib()
    for s in SYMBOLS:
        assert re.search(r"\b%s\s*\(" % s, txt), "not declared: " + s
        assert hasattr(L, s), "not exported: " + s


def test_summary_struct_matches_the_header():
    body = re.search(r"typedef struct \{(.*?)\} zmt_frame_index;", _header(), flags=re.S).group(1)
    fields = re.findall(r"(uint32_t|uint64_t)\s+(\w+);", body)
    ct = {"uint32_t": ctypes.c_uint32, "uint64_t": ctypes.c_uint64}
    assert [(n, ct[t]) for t, n in fields] == list(z.FrameIndex._fields_)
    assert ctypes.sizeof(z.FrameIndex) == 40


def test_profiling_id_follows_the_lz4_hc_block_kernel():
    ids = re.search(r"enum \{(.*?)\};", _header(), flags=re.S).group(1)
    names = [re.sub(r"\s*=.*", "", x).strip() for x in ids.split(",")]
    assert names.index("ZMT_K_FRAME_INDEX") == names.index("ZMT_K_L4H_BLOCKS") + 1 == 16
    assert names[-1] == "ZMT_K_COUNT"
