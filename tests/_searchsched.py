"""The parallel lazy parse of the chain-search encoders restated from best[] (plain Python and numpy).

zstd_lazy_blocks_kernel (zstd levels 6-12) parses each 16 KiB block as 256 ranges of 64 positions: nx[p] (the next free
position from p), ex[p] (the first position at or past the end of p's range that the parse reaches from p, resolved
backwards inside the range), the chained entries (the true parse's first position in each range), the fold flags of
entry matches that continue the sequence before them, and the carries those folds add to a sequence of an earlier
range.  lz4_hc_blocks_kernel (LZ4 levels 10-12) runs the same scheme over the four 16 KiB quarters of a 64 KiB block
and carries the parse position and one open sequence from one quarter into the next.

`zstd_block` and `lz4_block` return a block's sequences, (literal length, offset, match length), as the kernel builds
them, and the named events its schedule met; the tests compare the sequences with the CPU twins' and assert the events
each edge case is built for.  Events: a dict name -> list of details (one per occurrence)."""
from collections import defaultdict

import numpy as np

RANGE, QUARTER, LEN_BITS = 64, 16384, 9
LONGLIT = 32                               # C_LONGLIT: literal runs longer than this are queued as long jobs
LONG_ML_RUNS = 4                           # ... and match lengths whose 255-byte runs number more than this


def _len(m):
    return (m & ((1 << LEN_BITS) - 1)).astype(np.int64)


def _off(m):
    return (m >> LEN_BITS).astype(np.int64)


def _highbit(v):
    return (np.frexp(np.maximum(v, 1).astype(np.float64))[1] - 1).astype(np.int64)


def _zstd_gain(m):
    return 4 * _len(m) - _highbit(_off(m) + 3)


def _ranges(nx, nb, start):
    """ex[] per range, the chained entries (range -> position) and the position the chain leaves the block at."""
    nr = (nb + RANGE - 1) // RANGE
    ex = np.zeros(nb, np.int64)
    r0 = np.arange(nr) * RANGE
    r1 = np.minimum(r0 + RANGE, nb)
    for j in range(RANGE - 1, -1, -1):
        p = r0 + j
        ok = p < r1
        p, e = p[ok], r1[ok]
        x = nx[p]
        ex[p] = np.where(x >= e, x, ex[np.minimum(x, nb - 1)])
    entry, p = {}, start
    while p < nb:
        entry[p // RANGE] = p
        p = int(ex[p])
    return entry, p


def _next_match(nx, nb):
    """nm[p]: the first q >= p whose nx is not q + 1 (nb if none)."""
    idx = np.arange(nb)
    m = np.where(nx != idx + 1, idx, nb)
    return np.minimum.accumulate(m[::-1])[::-1] if nb else m


def _walk(nx, nm, off, e, r1):
    """The true parse of one range from its entry: (literal count, [(start, end, offset)] of its matches)."""
    lits, ms, p = 0, [], e
    while p < r1:
        q = min(int(nm[p]), r1)
        if q > p:
            lits += q - p
            p = q
            continue
        x = int(nx[p])
        ms.append((p, x, int(off[p])))
        p = x
    return lits, ms


def _schedule(nx, nm, off, nb, entry, fold, ev):
    """Walks 1 and 2 over the ranges of one parse unit.  fold: ranges whose entry match continues the sequence before
    them (set here for the entries that follow a range's last match; the caller may have set the unit's first).
    Returns per range (range, its new sequences [start, offset, merged length], carry, literal count, its matches)."""
    nr = (nb + RANGE - 1) // RANGE
    per = []
    for r in range(nr):
        r1 = min((r + 1) * RANGE, nb)
        if r not in entry:
            per.append(None)
            continue
        e = entry[r]
        lits, ms = _walk(nx, nm, off, e, r1)
        for p, x, o in ms:
            if x >= r1 and x < nb and nx[x] != x + 1 and off[x] == o:
                fold.add(x // RANGE)
        per.append((e, lits, ms))
    res = []
    for r in range(nr):
        if per[r] is None:
            res.append((r, [], 0, 0, []))
            continue
        e, lits, ms = per[r]
        efold = bool(ms) and ms[0][0] == e and r in fold
        seqs, carry, poff, cur = [], 0, 0, None
        q = e
        for p, x, o in ms:
            if p > q:
                poff = 0                                         # literals between
            if (efold if p == e else o == poff):
                if cur is not None:
                    cur[2] += x - p
                else:
                    carry += x - p
            else:
                cur = [p, o, x - p]
                seqs.append(cur)
            poff, q = o, x
        res.append((r, seqs, carry, lits, ms))
        if efold:
            ev["fold_at_entry"].append(e % RANGE)
    return res


def _range_events(nx, nb, entry, res, ev, base):
    nr = (nb + RANGE - 1) // RANGE
    for r in range(nr):
        if r not in entry:
            ev["range_no_entry"].append(base + r * RANGE)
        elif r and nx[entry[r]] == entry[r] + 1:
            ev["entry_is_literal"].append(base + entry[r])
    for r, seqs, carry, lits, ms in res:
        for p, x, o in ms:
            r1 = (p // RANGE + 1) * RANGE
            if x < nb and x % RANGE == 0:
                ev["match_ends_at_range_end"].append(base + x)
            if x < nb and x % RANGE == RANGE - 1:
                ev["match_ends_one_before_range_end"].append(base + x)
            if x < nb and x % RANGE == 1 and x > r1:
                ev["match_ends_one_past_range_end"].append(base + x)
            if x // RANGE - p // RANGE >= 2:
                ev["match_skips_range"].append(base + p)
        if carry and r and not res[r - 1][1]:
            ev["fold_after_range_without_sequence"].append(base + r * RANGE)


def _carry_sources(res, ev, open_before=0):
    """Adds each range's carry to the last sequence written before it; records how many ranges carried into each."""
    flat, src = [], []
    pending = defaultdict(int)
    for r, seqs, carry, lits, ms in res:
        if carry:
            tgt = len(flat) + open_before - 1
            assert tgt >= 0, "a carry with no sequence before it"
            pending[tgt] += 1
            src.append((tgt, carry))
        flat.extend(seqs)
    for k in pending.values():
        ev["carry_from_k_ranges"].append(k)
    return flat, src


def _deferrals(nx, best, nb, visited, look, unit, ev, name, base):
    """Visited positions with a match that the lazy rule turned into a literal because of a candidate in the next unit
    (range or quarter) of `unit` positions; detail (position, 1 or 2 positions ahead)."""
    p = np.flatnonzero((best[:nb] != 0) & (nx[:nb] == np.arange(nb) + 1) & visited[:nb])
    for q in p.tolist():
        k = look(q)
        if k and (q + k) // unit != q // unit:
            ev[name].append((base + q, k))


# ------------------------------------------------------------------------------------------------- zstd
def zstd_block(bb, lazy, ev=None, base=0):
    """The kernel's parse of one 16 KiB zstd block from its best[] (bb, length nb): [(ll, off, ml)], events."""
    ev = defaultdict(list) if ev is None else ev
    bb = np.asarray(bb, np.uint32)
    nb = int(bb.size)
    idx = np.arange(nb)
    z = np.zeros(2, np.uint32)
    b1, b2 = np.concatenate([bb[1:], z[:1]]), np.concatenate([bb[2:], z])
    g, g1, g2 = _zstd_gain(bb), _zstd_gain(b1), _zstd_gain(b2)
    d1 = (b1 != 0) & (g1 > g + 4)
    d2 = (lazy >= 2) & (b2 != 0) & (g2 > g + 7)
    nx = np.where((bb != 0) & ~d1 & ~d2, idx + _len(bb), idx + 1)
    off = _off(bb)
    entry, _ = _ranges(nx, nb, 0)
    nm = _next_match(nx, nb)
    fold = set()
    res = _schedule(nx, nm, off, nb, entry, fold, ev)
    _range_events(nx, nb, entry, res, ev, base)
    flat, carries = _carry_sources(res, ev)
    # literal lengths: the anchor entering a range is the largest match end of the ranges before it
    lend, anchor0 = 0, []
    for r, seqs, carry, lits, ms in res:
        anchor0.append(lend)
        if ms:
            lend = max(lend, ms[-1][1])
    out = []
    for (r, seqs, carry, lits, ms), a0 in zip(res, anchor0):
        anchor, ends = a0, {p: x for p, x, _ in ms}
        for p, x, o in ms:
            for s in seqs:
                if s[0] == p:
                    out.append([p - anchor, s[1], s[2]])
            anchor = x
    for tgt, carry in carries:
        out[tgt][2] += carry
    visited = _visited(nx, nm, entry, nb)
    _deferrals(nx, bb, nb, visited, lambda q: 1 if d1[q] else 2, RANGE, ev, "defer_looks_into_next_range", base)
    return [tuple(s) for s in out], ev


def _visited(nx, nm, entry, nb):
    """Positions the true parse stands on (literals and match starts)."""
    v = np.zeros(nb + 1, bool)
    p = min(entry.values()) if entry else nb
    while p < nb:
        q = int(nm[p])
        if q > p:
            v[p: q] = True
            p = q
        else:
            v[p] = True
            p = int(nx[p])
    return v


def zstd_chunk(best, lazy, block=16384):
    """Every block of one chunk: ([[(ll, off, ml)] per block], events)."""
    ev, out = defaultdict(list), []
    for b0 in range(0, int(best.size), block):
        s, _ = zstd_block(best[b0: b0 + block], lazy, ev, b0)
        out.append(s)
    return out, ev


# ------------------------------------------------------------------------------------------------- LZ4
def lz4_block(bb, lazy, ev=None, base=0):
    """The kernel's parse of one 64 KiB LZ4 block from its best[] (bb, length n): [(ll, off, ml)], events."""
    ev = defaultdict(list) if ev is None else ev
    bb = np.asarray(bb, np.uint32)
    n = int(bb.size)
    pad = np.concatenate([bb, np.zeros(2, np.uint32)])
    L = _len(pad)
    pos, open_, anchor, out = 0, None, 0, []
    for q0 in range(0, n, QUARTER):
        nb = min(QUARTER, n - q0)
        qb = pad[q0: q0 + nb]
        idx = np.arange(nb)
        l0, l1, l2 = L[q0: q0 + nb], L[q0 + 1: q0 + nb + 1], L[q0 + 2: q0 + nb + 2]
        d1 = l1 > l0 + 1
        d2 = (lazy >= 2) & (l2 > l0 + 2)
        nx = np.where((qb != 0) & ~d1 & ~d2, idx + l0, idx + 1)
        off = _off(qb)
        p0 = pos - q0
        assert 0 <= p0 < nb
        if p0:
            ev["quarter_carry_pos"].append(p0)
        fold = set()
        if open_ is not None:
            if nx[p0] == p0 + 1:
                ev["quarter_entry_literal"].append(base + pos)
            elif open_[0] + open_[2] == pos and open_[1] == off[p0]:
                fold.add(p0 // RANGE)
                ev["quarter_entry_fold"].append(p0)
            else:
                ev["quarter_entry_no_fold"].append(base + pos)
        entry, pend = _ranges(nx, nb, p0)
        nm = _next_match(nx, nb)
        res = _schedule(nx, nm, off, nb, entry, fold, ev)
        _range_events(nx, nb, entry, res, ev, base + q0)
        for r, seqs, carry, lits, ms in res:
            for s in seqs:
                s[0] += q0
        flat, carries = _carry_sources(res, ev, 1 if open_ is not None else 0)
        held = ([open_] if open_ is not None else []) + flat
        for tgt, carry in carries:
            held[tgt][2] += carry
        last = q0 + nb == n
        if not flat and open_ is not None and not last:
            ev["open_across_whole_quarter"].append(base + q0)
        ne = len(held) if last else max(len(held) - 1, 0)
        ev["held_sequences"].append(len(held))
        jobs = 0
        for s in held[:ne]:
            lit = s[0] - anchor
            out.append((lit, s[1], s[2]))
            jobs += lit > LONGLIT
            ml = s[2] - 4
            jobs += ml >= 15 and (ml - 15) // 255 > LONG_ML_RUNS
            anchor = s[0] + s[2]
        ev["long_jobs"].append(jobs)
        visited = _visited(nx, nm, entry, nb)
        _deferrals(nx, qb, nb, visited, lambda q: 1 if d1[q] else 2, RANGE, ev, "defer_looks_into_next_range", base + q0)
        _deferrals(nx, qb, nb, visited, lambda q: 1 if d1[q] else 2, nb, ev, "defer_looks_into_next_quarter", base + q0)
        open_ = held[-1] if held and not last else None
        pos = q0 + pend
    return out, ev


def lz4_chunk(best, lazy, block=65536):
    ev, out = defaultdict(list), []
    for b0 in range(0, int(best.size), block):
        s, _ = lz4_block(best[b0: b0 + block], lazy, ev, b0)
        out.append(s)
    return out, ev
