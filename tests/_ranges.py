"""The range-read rule (include/zstdmt_b200_dev.h, "Range reads"), restated in Python.

Content offsets come from the frames' own headers; a good range touches the frames from the first whose content ends
past its start to the last whose content starts before its end; every touched frame is selected once, in stream order;
the selected frames' content lies back to back in the scratch; dst_off is the prefix of the good ranges' lengths; a range
gets BAD_ARG, or the status of the first failed frame it touches, or OK."""
import bisect

import numpy as np

ST_OK, ST_BLOCK, ST_CONTENT_CHECKSUM, ST_CONTENT_SIZE, ST_UNSUPPORTED, ST_BAD_ARG = 0, 5, 7, 8, 10, 12
U64 = 1 << 64
PIECE = 64 * 1024


def rd(b, p, k):
    return int.from_bytes(bytes(b[p: p + k]), "little")


def lz4_content_size(frame):
    """The content size an LZ4F header states (FLG bit 3 + LE64 at 6), 0 for a frame without one whose first block header
    is the end mark (an empty input), or None."""
    if len(frame) < 7 or rd(frame, 0, 4) != 0x184D2204:
        return None
    if frame[4] & 8:
        return rd(frame, 6, 8) if len(frame) >= 15 else None
    h = 7 + (4 if frame[4] & 1 else 0)
    return 0 if len(frame) >= h + 4 and rd(frame, h, 4) == 0 else None


def zstd_content_size(frame):
    """Frame_Content_Size of a zstd frame header (RFC 8878 3.1.1.1.4), or None without one."""
    fhd = int(frame[4])
    fcs, single = fhd >> 6, (fhd >> 5) & 1
    pos = 5 + (0 if single else 1) + [0, 1, 2, 4][fhd & 3]
    n = [1 if single else 0, 2, 4, 8][fcs]
    if n == 0:
        return None
    v = rd(frame, pos, n)
    return v + 256 if n == 2 else v


def content_sizes(frames, codec):
    f = lz4_content_size if codec == "lz4" else zstd_content_size
    return [f(np.asarray(x, np.uint8)) for x in frames]


def content_table(sizes, csizes):
    """(status, bad frame, offsets): the exclusive prefix of the content sizes.  The first frame without a size fails
    the table with UNSUPPORTED, one stating more than 32768 bytes per compressed byte with CONTENT_SIZE."""
    off = [0]
    for f, (s, c) in enumerate(zip(sizes, csizes)):
        if s is None:
            return ST_UNSUPPORTED, f, None
        if s > int(c) * 32768:
            return ST_CONTENT_SIZE, f, None
        off.append(off[-1] + s)
    return ST_OK, len(sizes), off


def span(off, start, length):
    """The frames a good non-empty range touches, (first, last)."""
    fa = bisect.bisect_right(off, start, 1) - 1
    fb = bisect.bisect_right(off, start + length - 1, fa + 1) - 1
    return fa, fb


def is_bad(off, start, length):
    return start + length >= U64 or start + length > off[-1]


def plan(off, ranges, csize=None):
    """The plan of a batch: selected frames in stream order, each range's span (None: empty or bad), dst_off, the
    scratch offset of each selected frame, and (with the frames' compressed sizes) the packed bytes of the LZ4 read."""
    spans, sel, dst = [], set(), [0]
    for s, n in ranges:
        s, n = int(s) % U64, int(n) % U64
        bad = is_bad(off, s, n)
        sp = None if bad or n == 0 else span(off, s, n)
        if sp:
            sel.update(range(sp[0], sp[1] + 1))
        spans.append((bad, sp))
        dst.append(dst[-1] + (0 if bad else n))
    sel = sorted(sel)
    scr = [0]
    for f in sel:
        scr.append(scr[-1] + off[f + 1] - off[f])
    packed = sum(16 + (int(csize[f]) + 15) // 16 * 16 for f in sel) if csize is not None else None
    pieces = sum(-(-int(n) // PIECE) for (bad, sp), (_, n) in zip(spans, ranges) if sp)
    return dict(sel=sel, spans=spans, dst_off=dst, scratch_off=scr, packed=packed, pieces=pieces)


def apply(off, ranges, p, contents, frame_status=None):
    """Per-range (status, bytes) from the selected frames' decoded contents (contents[f] for f in p["sel"]) and their
    decode statuses: BAD_ARG, the first failed frame's status among those the range touches, or OK with its bytes."""
    scratch = np.concatenate([np.asarray(contents[f], np.uint8) for f in p["sel"]]) if p["sel"] else np.zeros(0, np.uint8)
    where = {f: i for i, f in enumerate(p["sel"])}
    out = []
    for (s, n), (bad, sp) in zip(ranges, p["spans"]):
        if bad:
            out.append((ST_BAD_ARG, None))
            continue
        if sp is None:
            out.append((ST_OK, np.zeros(0, np.uint8)))
            continue
        fail = [frame_status[f] for f in range(sp[0], sp[1] + 1) if frame_status and frame_status.get(f, ST_OK) != ST_OK]
        if fail:
            out.append((fail[0], None))
            continue
        a = p["scratch_off"][where[sp[0]]] + int(s) - off[sp[0]]
        out.append((ST_OK, scratch[a: a + int(n)]))
    return out


def ranges_for(off, rng, nrandom=10000, max_len=None):
    """The test range set over content offsets `off`: empty ranges (one at the end), 1 byte at each frame's first and last
    byte, ranges +-1 around every boundary, one over three or more frames, the whole content, duplicates and overlaps in
    unsorted order, and `nrandom` seeded random ranges."""
    total = off[-1]
    r = [(0, 0), (total, 0), (total // 2, 0)]
    for f in range(len(off) - 1):
        a, b = off[f], off[f + 1]
        if b > a:
            r += [(a, 1), (b - 1, 1)]
        if 0 < a < total:
            r += [(a - 1, 1), (a - 1, 2), (a, 1), (max(0, a - 2), min(4, total - max(0, a - 2)))]
    nonempty = [f for f in range(len(off) - 1) if off[f + 1] > off[f]]
    if len(nonempty) >= 3:
        a, b = off[nonempty[0] + 1] - 1, off[nonempty[2]] + 1
        r.append((a, b - a))
    r.append((0, total))
    dup = [r[i] for i in rng.integers(0, len(r), size=min(len(r), 32))]
    r += dup + [(s + n // 3, n - n // 3) for s, n in dup]
    max_len = max_len or max(1, total)
    st = rng.integers(0, total + 1, size=nrandom) if total else np.zeros(nrandom, np.int64)
    ln = np.minimum(rng.integers(0, max_len + 1, size=nrandom), total - st)
    r += list(zip(st.tolist(), ln.tolist()))
    perm = rng.permutation(len(r))
    return [r[i] for i in perm]
