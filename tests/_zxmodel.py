"""Models of two zstd decoder kernels (zstdmt_b200/csrc/zstd_decode.cu; the execute pass shares match_exec.cuh), so that the edges of their GPU schedules can be
named on the oracle's block trace (orc_zstd_trace) and on the frame's bytes.

exec_steps(trace, b) restates zx_block, the execute pass ("kernel 3"), on one compressed block: how its sequences are cut
into steps of at most STEP_CAP sequences and ZX_SPAN bytes (or a lone step for a first sequence larger than the span),
which path copies every literal run and every match, where each match's source lies, and whether the match is dependent.
Dependence is computed twice — the exact pairwise overlap with the earlier destinations of the step, and the kernel's
lower-bound search over lanes — and the two must agree.

lane_reader(frame, blk) restates FastBits and the decode loop of zstd_seq_predef_kernel on the block's sequence section:
per sequence, the bit phase at the refill, the valid bits, the extra bits read before the state updates, whether the
second refill fires, and the slack left before the next refill.

The constants below are the model's own; test_zstd_exec_model.py reads the kernel's from the source and compares."""
import os
import re
from collections import Counter

import numpy as np

ZX_SPAN = 2048          # bytes one execute step may regenerate (staged in shared memory)
STEP_CAP = 32           # sequences per execute step: one per lane
LANE_LIT = 32           # literal runs up to this length are copied by their own lane, longer ones by the warp
OWN_ML = 32             # independent matches up to this length are copied by their own lane
CHUNK = 32              # in-order copies with an offset below this are copied modulo the offset
REFILL_AT = 40          # the lane reader refills a second time when the extra bits of a sequence exceed this
OFC_MAX = 24            # larger offset codes send the block to the general sequence decoder
INACTIVE = 0x7FFFFFFF   # e_end / d_beg of lanes without a match in the kernel's search

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zstdmt_b200", "csrc")


def kernel_constants():
    """The same constants as the source states them.  Each use site is found by a regex (a missing match is an error)
    and must name its constant; the value is the constant's #define in match_exec.cuh (what the execute pass shares
    with the LZ4 decoder) or zstd_decode.cu."""
    from _searchcorpus import kernel_constant
    files = ("match_exec.cuh", "zstd_decode.cu")
    src = {f: open(os.path.join(CSRC, f)).read() for f in files}

    def one(f, pat):
        m = re.findall(pat, src[f])
        assert m, "pattern not found in %s: %s" % (f, pat)
        m = {tuple(int(x) if x.isdigit() else kernel_constant(x, files) for x in (v if isinstance(v, tuple) else (v,))) for v in m}
        assert len(m) == 1, (pat, m)
        v = m.pop()
        return v if len(v) > 1 else v[0]
    z, x = "zstd_decode.cu", "match_exec.cuh"
    cap = one(z, r"uint32_t cnt = B\.nseq - base < (\w+) \? B\.nseq - base : (\w+);")
    assert cap[0] == cap[1], cap
    return {
        "ZX_SPAN": one(z, r"lane < cnt && it <= (\w+)\)"),
        "STEP_CAP": cap[0],
        "LANE_LIT": one(z, r"if \(lane < lim && ll <= (\w+)\)"),
        "LANE_LIT_WARP": one(z, r"__ballot_sync\(0xFFFFFFFFu, lane < lim && ll > (\w+)\)"),
        "OWN_ML": one(z, r"if \(indep && ml <= (\w+)\)"),
        "OWN_ML_BALLOT": one(z, r"act && !\(indep && ml <= (\w+)\)"),
        "CHUNK": one(x, r"else if \(off >= (\w+)\)"),
        "REFILL_AT": one(z, r"if \(ofc \+ \(mx >> 24\) \+ \(lx >> 24\) > (\d+)\) R\.refill\(\);"),
        "OFC_MAX": one(z, r"if \(ofc > (\d+)\) return;"),
        "INACTIVE": one(x, r"e_end = act \? \(int32_t\)\(dst \+ ml\) : (\w+),"),
    }


# ---------------------------------------------------------------------------------------------------- the execute pass
def block_starts(tr):
    """Frame position of every block's first output byte (and the frame size at the end)."""
    return np.concatenate([[0], np.cumsum(tr.col("regen").astype(np.int64))])


def kernel_dependent(lane, sp, ml, d_beg, e_end):
    """The kernel's test: a = lower bound of e_end <= sp over the 32 lanes by a 5-step shuffle search, then
    a < lane && d_beg[a] < sp + ml.  d_beg / e_end: 32 entries, INACTIVE for lanes without a match."""
    a = 0
    for stp in (16, 8, 4, 2, 1):
        if e_end[(a + stp - 1) & 31] <= sp:
            a += stp
    return a < lane and d_beg[a & 31] < sp + ml


def _form(off, ml):
    return "straight" if off >= ml else ("chunk32" if off >= CHUNK else "modulo")


def exec_steps(tr, b, starts=None):
    """zx_block on compressed block b of the trace.  Returns {"steps", "seqs", "trailing", "events"}:
    steps: kind ("step" | "lone"), op and lp at the step start, span (bytes), end ("cap" | "span" | "end"), first
           (index of its first sequence in the block) and n (sequences);
    seqs:  per sequence step, lane, op (literal start), mp (match start), ll, off, ml, lit ("lane" | "warp"), match
           ("own" | "inorder" | "lone"), form (copy form of in-order and lone matches), nlow (own-lane matches), where
           ("window" | "below" | "earlier"), back (blocks back, earlier-block sources), straddle (an earlier-block source
           that reaches into this block), dep (pairwise) and dep_kernel (the kernel's search), indep;
    trailing: the block's literals after the last sequence; events: a Counter of named edges."""
    if starts is None:
        starts = block_starts(tr)
    types = tr.col("type")
    q = tr.block_seqs(b).astype(np.int64)
    n = len(q)
    rg, lreg = int(tr.blk[b, 3]), int(tr.col("lit_regen")[b])
    blk0 = int(starts[b])
    ev, steps, seqs = Counter(), [], []
    op = lp = base = 0
    inorder_dest = []                                     # (start, end) of in-order matches of earlier steps of the block

    def where(sp, ml, rec, op):
        if sp >= op:
            rec["where"] = "window"
        elif sp >= 0:
            rec["where"] = "below"
        else:
            rec["where"] = "earlier"
            src_blk = int(np.searchsorted(starts, blk0 + sp, side="right") - 1)
            rec["back"] = b - src_blk
            rec["straddle"] = sp + ml > 0
            path = rec["match"]
            ev["cross_%s_back%d" % (path, min(rec["back"], 3))] += 1
            if rec["straddle"]:
                ev["cross_%s_straddle" % path] += 1
            ev["cross_first_step" if op == 0 else "cross_later_step"] += 1
            between = {int(t) for t in types[src_blk: b]}
            if 0 in between:
                ev["cross_over_raw"] += 1
            if 1 in between:
                ev["cross_over_rle"] += 1

    prev_lone = None
    while base < n:
        cnt = min(n - base, STEP_CAP)
        sizes = q[base: base + cnt, 0] + q[base: base + cnt, 2]
        tot = np.cumsum(sizes)
        nfit = int((tot <= ZX_SPAN).sum())
        if nfit == 0:                                       # lone: the first sequence alone exceeds the span
            ll, off, ml = int(q[base, 0]), int(q[base, 3]), int(q[base, 2])
            mp = op + ll
            end = "end" if base + 1 == n else "span"
            steps.append(dict(kind="lone", op=op, lp=lp, span=ll + ml, end=end, first=base, n=1))
            rec = dict(step=len(steps) - 1, lane=0, op=op, mp=mp, ll=ll, off=off, ml=ml, lit="warp", match="lone",
                       form=_form(off, ml), nlow=None, dep=None, dep_kernel=None, indep=None)
            where(mp - off, ml, rec, op)
            seqs.append(rec)
            ev["lone_" + rec["form"]] += 1
            if ml > ZX_SPAN and off in (1, 2, 3, 31, 32, 33):
                ev["lone_off_%d" % off] += 1
            if ml > ZX_SPAN and off >= ml:
                ev["lone_straight_long"] += 1
            if ll > ZX_SPAN and mp - off >= op:
                ev["lone_reads_own_literals"] += 1
            if base == 0:
                ev["lone_first"] += 1
            if base + 1 == n:
                ev["lone_last"] += 1
            if rec["form"] != "straight":
                inorder_dest.append((mp, mp + ml))
            prev_lone = (op, op + ll + ml)
            op += ll + ml; lp += ll; base += 1
            continue
        ll, off, ml = q[base: base + nfit, 0], q[base: base + nfit, 3], q[base: base + nfit, 2]
        span = int(tot[nfit - 1])
        if base + nfit == n:
            end = "end"
        elif nfit == STEP_CAP:
            end = "cap"
        else:
            end = "span"
        steps.append(dict(kind="step", op=op, lp=lp, span=span, end=end, first=base, n=nfit))
        ev["step_" + end] += 1
        if end == "span":
            if span == ZX_SPAN:
                ev["step_span_2048"] += 1
            if span + int(sizes[nfit]) == ZX_SPAN + 1:
                ev["step_span_2049"] += 1
        if nfit == 1 and span == ZX_SPAN:
            ev["step_single_2048"] += 1
        my_op = op + tot[:nfit] - (ll + ml)
        mp = my_op + ll
        sp = mp - off
        e_end = [int(x) for x in mp + ml] + [INACTIVE] * (32 - nfit)
        d_beg = [int(x) for x in mp] + [INACTIVE] * (32 - nfit)
        recs = []
        for i in range(nfit):
            li, oi, mi, s = int(ll[i]), int(off[i]), int(ml[i]), int(sp[i])
            dep = bool(((mp[:i] < s + mi) & (s < mp[:i] + ml[:i])).any())
            depk = kernel_dependent(i, s, mi, d_beg, e_end)
            assert dep == depk, ("the kernel's dependency search differs from the pairwise overlap", b, base + i)
            indep = oi >= mi and not dep
            own = indep and mi <= OWN_ML
            rec = dict(step=len(steps) - 1, lane=i, op=int(my_op[i]), mp=int(mp[i]), ll=li, off=oi, ml=mi,
                       lit="lane" if li <= LANE_LIT else "warp", match="own" if own else "inorder",
                       form=None if own else _form(oi, mi), dep=dep, dep_kernel=depk, indep=indep,
                       nlow=(0 if s >= op else min(op - s, mi)) if own else None)
            where(s, mi, rec, op)
            recs.append(rec)
            # literal paths
            if li <= LANE_LIT:
                ev["lit_lane_%d" % li] += 1
            else:
                ev["lit_warp_33" if li == LANE_LIT + 1 else "lit_warp_long"] += 1
            # match paths
            if own:
                ev["own"] += 1
                ev["nlow_%d_%d" % (mi, rec["nlow"])] += 1
                if oi == mi:
                    ev["own_off_eq_ml_%d" % mi] += 1
                if mi == OWN_ML:
                    ev["indep_own_32"] += 1
            else:
                ev["inorder_" + rec["form"]] += 1
                if oi == mi - 1 and mi <= OWN_ML:
                    ev["inorder_off_ml_minus_1_%d" % mi] += 1
                if indep and mi == OWN_ML + 1:
                    ev["indep_inorder_33"] += 1
            # dependency boundaries against every earlier destination of the step
            for j in range(i):
                dj, ej = int(mp[j]), int(mp[j] + ml[j])
                if s + mi == dj:
                    ev["dep_src_end_at_dest"] += 1
                if s + mi == dj + 1:
                    ev["dep_src_end_one_into_dest"] += 1
                    if recs[j]["match"] == "inorder":
                        ev["dep_src_end_one_into_inorder_dest"] += 1
                if s == ej:
                    ev["dep_src_start_at_dest_end"] += 1
                if s == ej - 1:
                    ev["dep_src_start_one_before_dest_end"] += 1
                if recs[j]["match"] == "inorder" and dj < s + mi and s < ej:
                    ev["inorder_reads_inorder" if not own else "own_reads_inorder_same_step"] += 1
            # literal runs of this step read back through the window
            for j in range(i + 1):
                a0, a1 = int(my_op[j]), int(my_op[j] + ll[j])
                if a0 < a1 and a0 < s + mi and s < a1:
                    ev["reads_%s_literals" % recs[j]["lit"]] += 1
            if own and any(d0 < s + mi and s < d1 for d0, d1 in inorder_dest):
                ev["own_reads_earlier_inorder"] += 1
            if prev_lone is not None and prev_lone[0] < s + mi and s < prev_lone[1]:
                ev["lone_read_next"] += 1
        if nfit == STEP_CAP and all(r["dep"] for r in recs[1:]):
            ev["dep_chain_31"] += 1
        for r in recs:
            if r["match"] == "inorder":
                inorder_dest.append((r["mp"], r["mp"] + r["ml"]))
        seqs += recs
        prev_lone = None
        op += span; lp += int(ll.sum()); base += nfit
    trailing = lreg - lp
    assert trailing >= 0 and op + trailing == rg, ("steps and trailing literals do not regenerate the block", b)
    ev["trailing_%s" % (trailing if trailing <= 1 else "ge33" if trailing > LANE_LIT else "2_32")] += 1
    return dict(steps=steps, seqs=seqs, trailing=trailing, events=ev)


def exec_frame(tr):
    """exec_steps over every compressed block with sequences: ({block: result}, events of the frame)."""
    starts, out, ev = block_starts(tr), {}, Counter()
    for b in np.flatnonzero((tr.col("type") == 2) & (tr.col("nseq") > 0)):
        r = exec_steps(tr, int(b), starts)
        out[int(b)] = r
        ev += r["events"]
    return out, ev


# ---------------------------------------------------------------------------------------------------- the lane reader
# predefined distributions and length codes of RFC 8878 (section 3.1.1.3.2.2)
LL_NORM = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_NORM = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_NORM = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_BASE = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512,
           1024, 2048, 4096, 8192, 16384, 32768, 65536]
ML_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31,
           32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539]


def fse_table(norm, log):
    """FSE decoding table of a normalized distribution (RFC 8878 4.1.1): per state (symbol, nbBits, baseline)."""
    size = 1 << log
    high, sym, nxt = size - 1, [0] * size, [0] * len(norm)
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s; high -= 1; nxt[s] = 1
        else:
            nxt[s] = c
    step, pos = (size >> 1) + (size >> 3) + 3, 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    out = []
    for u in range(size):
        s = sym[u]; x = nxt[s]; nxt[s] += 1
        nb = log - (x.bit_length() - 1)
        out.append((s, nb, (x << nb) - size))
    return out


T_LL, T_ML, T_OF = fse_table(LL_NORM, 6), fse_table(ML_NORM, 6), fse_table(OF_NORM, 5)


def frame_blocks(frame):
    """Walk one zstd frame: ([(block type, offset of the block's content in the frame, content bytes)], needs_seq),
    needs_seq as the host scan flags it: some block has treeless literals or a sequence table that is not predefined."""
    f = np.ascontiguousarray(frame, dtype=np.uint8)
    assert int.from_bytes(f[:4].tobytes(), "little") == 0xFD2FB528
    fhd = int(f[4]); single = (fhd >> 5) & 1
    pos = 5 + (0 if single else 1) + (0, 1, 2, 4)[fhd & 3] + ((1 if single else 0), 2, 4, 8)[fhd >> 6]
    out, needs = [], False
    while True:
        h = int(f[pos]) | int(f[pos + 1]) << 8 | int(f[pos + 2]) << 16
        typ, size = (h >> 1) & 3, h >> 3
        clen = 1 if typ == 1 else size
        out.append((typ, pos + 3, clen))
        if typ == 2:
            s = _sections(f[pos + 3: pos + 3 + clen])
            if s["ltype"] == 3 or (s["nseq"] > 0 and s["modes"] != 0):
                needs = True
        pos += 3 + clen
        if h & 1:
            return out, needs


def _sections(src):
    """Literals and sequences section headers of a compressed block, read as zstd_seq_predef_kernel reads them."""
    b0 = int(src[0]); lt, sf = b0 & 3, (b0 >> 2) & 3
    if lt < 2:
        lhdr = (1, 2, 1, 3)[sf]
        lregen = b0 >> 3 if sf in (0, 2) else (b0 >> 4) | int(src[1]) << 4 | ((int(src[2]) << 12) if sf == 3 else 0)
        lcomp = lregen if lt == 0 else 1
    else:
        v = int.from_bytes(src[:5].tobytes(), "little")
        lhdr, lcomp = ((3, (v >> 14) & 0x3FF), (3, (v >> 14) & 0x3FF), (4, (v >> 18) & 0x3FFF), (5, (v >> 22) & 0x3FFFF))[sf]
    q = lhdr + lcomp
    q0 = int(src[q])
    if q0 < 128:
        nseq, used = q0, 1
    elif q0 < 255:
        nseq, used = ((q0 - 128) << 8) + int(src[q + 1]), 2
    else:
        nseq, used = int(src[q + 1]) + (int(src[q + 2]) << 8) + 0x7F00, 3
    modes = int(src[q + used]) if nseq else -1
    return dict(ltype=lt, nseq=nseq, modes=modes, seq_start=q + used + 1)


def lane_reader(frame, b, addr=0, blocks=None):
    """FastBits and the decode loop of zstd_seq_predef_kernel on block b of the frame, whose first byte lies at input
    address `addr` (mod 8 is what matters).  None for blocks the kernel leaves to the general path: not compressed, in a
    frame the host scan flags, tables not all predefined, an offset code above OFC_MAX, a repeat Offset_Value (<= 3).
    Otherwise {"seqs": per sequence (ll, Offset_Value, ml, bitpos at the refill, V, S1, refill2, slack, state bits),
    "section": the sequence section's start address mod 8, "nbytes": bitstream bytes, "events": Counter}."""
    f = np.ascontiguousarray(frame, dtype=np.uint8)
    if blocks is None:
        blocks = frame_blocks(f)
    bl, needs = blocks
    typ, coff, clen = bl[b]
    if typ != 2 or needs:
        return None
    src = f[coff: coff + clen]
    s = _sections(src)
    if s["nseq"] == 0 or s["modes"] != 0:
        return None
    start = coff + s["seq_start"]
    stream = src[s["seq_start"]:]
    nbytes = len(stream)
    last = int(stream[-1])
    bitpos = nbytes * 8 - (8 - last.bit_length() + 1)
    ev = Counter()
    ev["section_mod8_%d" % ((addr + start) % 8)] += 1
    if nbytes <= 16:
        ev["short_stream"] += 1
    st = dict(bitpos=bitpos, base=0, win_top=0)

    def refill():
        bp = st["bitpos"]
        tb = (bp + 7) >> 3 if bp > 0 else 0
        b0 = tb - 8
        if b0 >= 0 and tb + 8 <= nbytes:
            ev["refill_aligned" if (addr + start + b0) % 8 == 0 else "refill_funnel"] += 1
        else:
            ev["refill_bytes"] += 1
        st["base"] = b0 * 8
        return bp - b0 * 8                                  # valid bits in the window

    padded = bytes(8) + stream.tobytes()                   # bits below the stream start read as zeros

    def read(nb):
        st["bitpos"] -= nb
        lo = st["bitpos"]
        assert lo >= st["base"], "read below the refilled window"
        p = lo + 64
        return (int.from_bytes(padded[p >> 3: (p >> 3) + 5], "little") >> (p & 7)) & ((1 << nb) - 1)

    refill()
    sLL, sOF, sML = read(6), read(5), read(6)
    out = []
    for i in range(s["nseq"]):
        bp = st["bitpos"]
        V = refill()
        top = bp
        llc, llb, llbase = T_LL[sLL]; mlc, mlb, mlbase = T_ML[sML]; ofc, ofb, ofbase = T_OF[sOF]
        if ofc > OFC_MAX:
            return None
        ofv = (1 << ofc) + read(ofc)
        ml = ML_BASE[mlc] + read(ML_BITS[mlc])
        ll = LL_BASE[llc] + read(LL_BITS[llc])
        if ofv <= 3:
            return None
        s1 = ofc + ML_BITS[mlc] + LL_BITS[llc]
        r2, sb = False, 0
        if i + 1 < s["nseq"]:
            if s1 > REFILL_AT:
                r2 = True
                V2 = refill()
                top = st["bitpos"]; V = V2
                ev["second_refill"] += 1
            sb = llb + mlb + ofb
            sLL = llbase + read(llb); sML = mlbase + read(mlb); sOF = ofbase + read(ofb)
        slack = V - (top - st["bitpos"])
        assert st["bitpos"] >= 0, "bit stream exhausted"
        out.append(dict(ll=ll, ofv=ofv, ml=ml, bitpos=bp, V=56 + bp % 8 if bp % 8 else 64, S1=s1, refill2=r2, slack=slack,
                        state=sb))
        if s1 in (40, 41):
            ev["s1_%d_phase%d" % (s1, bp % 8)] += 1
        if s1 == 55:
            ev["s1_55"] += 1
        if slack == 0:
            ev["slack_0"] += 1
        if s1 == REFILL_AT and sb == 17 and (56 + bp % 8 if bp % 8 else 64) == 57:
            ev["s1_40_v57_full_states"] += 1
    assert st["bitpos"] == 0, "bit stream not consumed exactly"
    return dict(seqs=out, section=(addr + start) % 8, nbytes=nbytes, events=ev)


def lane_frame(frame, addr=0):
    """lane_reader over every block of the frame: ({block: result}, events of the frame)."""
    blocks = frame_blocks(frame)
    out, ev = {}, Counter()
    for b in range(len(blocks[0])):
        r = lane_reader(frame, b, addr, blocks)
        if r is not None:
            out[b] = r
            ev += r["events"]
    return out, ev
