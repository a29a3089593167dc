"""A model of how z_encode_block (zstdmt_b200/csrc/zstd_entropy.cuh) spreads one block's entropy coding over its 256
threads, run on the trace of the entropy stage's CPU twin (_zenc.block_b200 with chains=True).  It restates literally
what the kernel does in parallel and checks that it gives the twin's serial results:
  - the FSE state chains (warp 7): c = ceil(nseq / 32) steps per lane, lanes past nseq idle, each lane's entry state
    guessed by a warm-up from init_state(codes[w0]) over the Z_WARM steps before its chunk (exact when the warm-up
    reaches step 0), then the repair loop as written: every round, each lane whose entry state differs from its
    predecessor's current exit re-runs from that exit, until no lane does; the final states are read from lane
    (nseq - 1) / c.  The kernel's claim, same bits as the serial chain, is asserted on every block;
  - the Huffman streams (warps 0-6): 4 groups of 56 threads, thread u of group k codes literals [a, b) of stream k at
    bit pos_lo of the stream, after everything that follows it; runs share their first and last words; the end marker
    sits at the stream's bit total, which gives sbytes and swords;
  - the sequence bits (all 256 threads): runs of g = ceil(nseq / 256) sequences each, placed by an exclusive scan.
events(trace) returns the named events of one block (a dict name -> value or count); the corpus's predicates use them."""
import numpy as np

import _zenc as ze
from _searchcorpus import kernel_constant
from _zxmodel import LL_BITS, ML_BITS

ENT = ("zstd_entropy.cuh",)
Z_WARM, Z_BITWORDS, Z_HUF_MAXBITS, Z_MAXSEQ, Z_MAXLIT = 16, 3072, 11, 4352, 64 * 1024 + 256
LANES, LIT_THREADS, GROUP, NT = 32, 224, 56, 256


def kernel_constants():
    """The #defines of zstd_entropy.cuh that the model restates."""
    return {n: kernel_constant(n, ENT) for n in ("Z_WARM", "Z_BITWORDS", "Z_HUF_MAXBITS", "Z_MAXSEQ", "Z_MAXLIT")}


_TABLES = {}


def table(k):
    """Encoder view of the predefined table of stream k: (size, init[s], step(state, s) -> state), states as the kernel
    holds them (size + cell)."""
    if k not in _TABLES:
        log, sym, nb, base = ze.fse_table(k)
        size = 1 << log
        nxt = np.full((64, size), -1, np.int64)                      # nxt[s, x]: the cell of s whose range holds x
        first = np.full(64, -1, np.int64)
        for u in range(size):
            s = sym[u]
            nxt[s, base[u]: base[u] + (1 << nb[u])] = u
            if first[s] < 0:
                first[s] = u
        _TABLES[k] = (size, nxt, first, nb)
    return _TABLES[k]


def init_state(k, s):
    size, _, first, _ = table(k)
    return size + int(first[s])


def step(k, st, s):
    size, nxt, _, _ = table(k)
    return size + int(nxt[s, st - size])


def chain_model(k, codes, serial, ev):
    """Warp 7 on stream k: the speculative chunks and the repair loop.  codes / serial: the twin's codes and serial states
    in encoding order."""
    n = len(codes)
    c = (n + LANES - 1) // LANES
    tb = [min(l * c, n) for l in range(LANES)]
    te = [min(t + c, n) for t in tb]
    have = [t < n for t in tb]

    def run(l, st):
        for t in range(tb[l], te[l]):
            st = init_state(k, codes[t]) if t == 0 else step(k, st, codes[t])
        return st

    sin, exact = [0] * LANES, [False] * LANES
    for l in range(LANES):
        if have[l]:
            w0 = tb[l] - Z_WARM if tb[l] > Z_WARM else 0
            st = init_state(k, codes[w0])
            for t in range(w0 + 1, tb[l]):
                st = step(k, st, codes[t])
            sin[l], exact[l] = st, w0 == 0
    sout = [run(l, sin[l]) if have[l] else 0 for l in range(LANES)]
    wrong0 = [l for l in range(1, LANES) if have[l] and sin[l] != serial[tb[l] - 1]]
    rounds, reruns, from_wrong = 0, [0] * LANES, 0
    while True:
        prev = [sout[l - 1] if l else sout[0] for l in range(LANES)]
        bad = [have[l] and l > 0 and prev[l] != sin[l] for l in range(LANES)]
        if not any(bad):
            break
        rounds += 1
        assert rounds <= LANES, "repair loop does not converge"
        for l in range(LANES):
            if bad[l]:
                from_wrong += prev[l] != serial[tb[l] - 1]
                sin[l] = prev[l]; sout[l] = run(l, sin[l]); reruns[l] += 1
    for l in range(LANES):                                           # the kernel comment's claim: the serial chain's states
        if have[l]:
            assert l == 0 or sin[l] == serial[tb[l] - 1], ("entry state", k, l)
            assert sout[l] == serial[te[l] - 1], ("exit state", k, l)
    fin_lane = (n - 1) // c
    assert sout[fin_lane] == serial[n - 1]
    name = "LL OF ML".split()[k]
    ev["lanes_busy"] = sum(have)
    ev["lanes_exact"] = sum(1 for l in range(LANES) if have[l] and exact[l])
    ev["spec_wrong_" + name] = len(wrong0)
    ev["repair_rounds_" + name] = rounds
    ev["rerun_twice_" + name] = sum(1 for r in reruns if r >= 2)
    ev["rerun_from_wrong_" + name] = from_wrong
    ev["fin_lane"] = fin_lane


def huffman_model(t, ev):
    """Warps 0-6 placing the four Huffman streams of a Huffman-coded literal section."""
    lits, hlen = np.asarray(t.lits, np.int64), t.hlen.astype(np.int64)
    nlit = len(lits)
    per = (nlit + 3) // 4
    bits = hlen[lits]
    run = []                                                         # (k, u, a, b, mybits)
    for tid in range(LIT_THREADS):
        k, u = divmod(tid, GROUP)
        s0 = k * per
        s1 = min(s0 + per, nlit)
        cnt = max(s1 - s0, 0)
        g = (cnt + GROUP - 1) // GROUP
        a = min(s0 + u * g, s1)
        b = min(a + g, s1)
        run.append((k, u, a, b, int(bits[a:b].sum())))
    pre = np.concatenate([[0], np.cumsum([r[4] for r in run])])
    sb = [int(pre[k * GROUP]) for k in range(4)] + [int(pre[-1])]
    tq = [sb[q + 1] - sb[q] for q in range(4)]
    assert tq == list(t.huf_bits), (tq, t.huf_bits)
    sbytes = [x // 8 + 1 for x in tq]
    swords = [(x + 32) // 32 for x in tq]
    assert sum(swords) <= Z_BITWORDS
    words = [dict() for _ in range(4)]                               # per stream: word -> threads that write it
    ends = [0] * 4
    for tid, (k, u, a, b, mb) in enumerate(run):
        pos_lo = sb[k + 1] - (int(pre[tid]) + mb)                    # after everything that follows the run in its stream
        if b > a:
            assert pos_lo == sb[k + 1] - sb[k] - ends[k] - mb        # the runs tile the stream, first literals on top
            ends[k] += mb
            for w in range(pos_lo >> 5, ((pos_lo + mb - 1) >> 5) + 1):
                words[k].setdefault(w, set()).add(tid)
    assert ends == tq
    shared = 0
    for k in range(4):
        shared += sum(1 for ts in words[k].values() if len(ts) > 1)
    # an 11-bit code across a word boundary in a word another run writes too
    straddle_shared = 0
    for tid, (k, u, a, b, mb) in enumerate(run):
        pos_lo = sb[k + 1] - (int(pre[tid]) + mb)
        p = pos_lo
        for i in range(b - 1, a - 1, -1):
            ln = int(bits[i])
            w0, w1 = p >> 5, (p + ln - 1) >> 5
            if ln == Z_HUF_MAXBITS and w0 != w1 and (len(words[k].get(w0, ())) > 1 or len(words[k].get(w1, ())) > 1):
                straddle_shared += 1
            p += ln
    ev["huf_nlit_mod4"] = nlit % 4
    ev["huf_empty_runs"] = sum(1 for r in run if r[3] == r[2])
    ev["huf_min_stream_lits"] = min(min((k + 1) * per, nlit) - min(k * per, nlit) for k in range(4))
    ev["huf_bits_mod8_0"] = sum(1 for x in tq if x % 8 == 0)
    ev["huf_bits_mod32_31"] = sum(1 for x in tq if x % 32 == 31)
    ev["huf_shared_words"] = shared
    ev["huf_straddle11_shared"] = straddle_shared
    ev["huf_sbytes"], ev["huf_swords"] = sbytes, swords


def seq_model(t, ev):
    """All 256 threads counting and placing the sequence bits: runs of g sequences in encoding order."""
    n = t.nseq
    g = (n + NT - 1) // NT
    rows = t.rows
    per = np.zeros(n, np.int64)
    for j in range(n):                                               # encoding order: j encodes sequence n-1-j
        ll, off, ml = (int(x) for x in rows[n - 1 - j])
        lc, oc, mc = (int(t.codes[k][j]) for k in range(3))
        b = LL_BITS[lc] + ML_BITS[mc] + oc
        if j:
            for k in range(3):
                size, _, _, nb = table(k)
                b += int(nb[int(t.states[k][j]) - size])
        per[j] = b
    runs = [(min(tid * g, n), min(tid * g + g, n)) for tid in range(NT)]
    tot = sum(int(per[a:b].sum()) for a, b in runs) + 17
    assert tot == t.seq_bits, (tot, t.seq_bits)
    ev["seq_threads_busy"] = sum(1 for a, b in runs if b > a)
    ev["seq_per_thread"] = g


def events(t):
    """The named events of one block, from the twin's trace (block_b200(..., chains=True))."""
    ev = {"nseq": t.nseq, "nlit": t.nlit, "regen": t.regen, "raw_reason": t.raw_reason, "lit_mode": t.lit_mode,
          "lit_reason": t.lit_reason, "est": t.est, "bsize": t.bsize, "seq_body": t.seq_body, "maxsym": t.maxsym,
          "wdesc_len": t.wdesc_len, "tree_bytes": t.tree_bytes}
    if t.nseq:
        for k in range(3):
            chain_model(k, t.codes[k], t.states[k], ev)
        seq_model(t, ev)
        ev["lls"] = set(int(x) for x in t.rows[:, 0])
    if t.lit_mode == 2:
        huffman_model(t, ev)
    return ev


def chunk_events(content, level):
    """[(block index, events)] of every block of one chunk."""
    out = []
    for b, (rows, lits, raw, last) in enumerate(ze.chunk_blocks(content, level)):
        _, t = ze.block_b200(rows, lits, raw, last, chains=True)
        out.append((b, events(t)))
    return out
