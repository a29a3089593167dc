"""Generate tests/golden/*.bin with the REAL reference (oracle/_ref: unmodified
lib/{lz4,zstd}-mt_*.c + liblz4 1.9.4 / libzstd 1.5.5).  Needs the reference tree at oracle
build time (oracle/Makefile REF); the fixtures are committed, so the suite does not."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _oracle as o
import zstdmt_b200 as z

CASES = [
    # codec, level, kind, n, chunk, first
    ("lz4", 1, z.GEN_MIX, 3 * 65536 + 17, 65536 * 2, 0),
    ("lz4", 1, z.GEN_TEXT, 150000, 1 << 20, 0),
    ("lz4", 3, z.GEN_MIX, 2 * 70000, 70000, 4),
    ("lz4", 1, z.GEN_ZEROS, 1 << 20, 1 << 20, 0),
    ("lz4", 1, z.GEN_MIX, 0, 1 << 20, 0),
    ("zstd", 3, z.GEN_TEXT, 200000, 1 << 20, 0),
    ("zstd", 3, z.GEN_MIX, 3 * 65536 + 5, 65536, 2),
    ("zstd", 1, z.GEN_MIX, 131072 * 2 + 9, 1 << 20, 5),
    # Small streams of what the suite otherwise only checks against a live reference build.  zstd level 19, mix class 2, one
    # two-block frame: block 0 has FSE-described sequence tables, block 1 treeless literals and Repeat_Mode tables (both
    # only legal after a first block).  LZ4 level 9, mix class 7: one frame of two linked blocks (FLG 0x4C).  Random bytes:
    # raw zstd blocks / stored LZ4 blocks.  Zeros: RLE zstd blocks.
    ("zstd", 19, z.GEN_MIX, 131072 + 512, 1 << 20, 2),
    ("zstd", 3, z.GEN_RANDOM, 2 * 1024 + 99, 1024, 0),
    ("zstd", 1, z.GEN_ZEROS, 3 * 16384 + 999, 16384, 0),
    ("lz4", 9, z.GEN_MIX, 65536 + 8192, 1 << 20, 7),
    ("lz4", 1, z.GEN_RANDOM, 2 * 1024 + 99, 1024, 0),
]

man = {"generator": "tests/golden/make_golden.py", "cases": []}
for i, (codec, level, kind, n, chunk, first) in enumerate(CASES):
    src = z.gen_stream(kind, n, chunk, first=first)
    rc, framed, st = o.ref_compress(o.CODEC_LZ4 if codec == "lz4" else o.CODEC_ZSTD, src, threads=2, level=level, chunk=chunk)
    assert rc == 0
    name = "%s_l%d_k%d_%d.bin" % (codec, level, kind, n)
    framed.tofile(os.path.join(HERE, name))
    man["cases"].append({"file": name, "codec": codec, "level": level, "kind": kind, "n": n, "chunk": chunk, "first": first,
                         "frames": int(st[1]), "framed_bytes": int(framed.size), "xxh32_framed": int(o.xxh32(framed)),
                         "xxh32_src": int(o.xxh32(src))})
with open(os.path.join(HERE, "manifest.json"), "w") as f:
    json.dump(man, f, indent=1)
print("wrote", len(CASES), "fixtures")
