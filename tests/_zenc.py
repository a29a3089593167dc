"""Plain-Python restatement of the choices the GPU zstd encoder (lz4_kernels.cu zstd_blocks_kernel, zstd_entropy.cuh)
makes on top of the LZ77 parse it shares with the LZ4 compressor (lz4_pipe.cuh), for tests that hold its output to them:
  - the parse: the LZ4 sequences of the bit-exact CPU twin orc_lz4_block_compress_b200 on the same 64 KiB window;
  - the sub-block cut: every 4 tiles (16 KiB) a block is closed at the start of the match still pending there;
  - the Huffman code: two-queue tree, length-limited to 11 bits (huf_lengths).
"""
import numpy as np

import _oracle as o

WINDOW = 65536
SUB = 4 * 4096                   # a sub-block is closed every 4 tiles of 4096 positions
HUF_MAXBITS = 11


def lz4_twin_block(win):
    """The CPU twin's LZ4 block for one window."""
    win = np.ascontiguousarray(win, dtype=np.uint8)
    L = o.orc()
    cap = L.orc_lz4_block_bound(win.size)
    out = np.empty(cap, np.uint8)
    n = L.orc_lz4_block_compress_b200(win.ctypes.data, win.size, out.ctypes.data, cap)
    return out[:n]


def lz4_sequences(block):
    """(match start, offset, match length) of every sequence of an LZ4 block, as an (n, 3) int64 array."""
    b = block.tobytes()
    i, pos, n, seqs = 0, 0, len(b), []
    while i < n:
        tok = b[i]; i += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                x = b[i]; i += 1; ll += x
                if x != 255:
                    break
        i += ll; pos += ll
        if i >= n:
            break                                   # the last sequence carries literals only
        off = b[i] | (b[i + 1] << 8); i += 2
        ml = tok & 15
        if ml == 15:
            while True:
                x = b[i]; i += 1; ml += x
                if x != 255:
                    break
        ml += 4
        seqs.append((pos, off, ml)); pos += ml
    return np.array(seqs, dtype=np.int64).reshape(-1, 3)


def sub_blocks(seqs, n):
    """Start positions of the sub-blocks of a window of n bytes whose twin parse is `seqs`: at 16, 32 and 48 KiB (when the
    window goes on) the encoder closes a block at the start of the last match that began before that point."""
    starts, z_pos = [0], 0
    for t1 in range(SUB, n, SUB):
        before = seqs[seqs[:, 0] < t1, 0] if len(seqs) else np.zeros(0, np.int64)
        c = int(before[-1]) if before.size else t1
        if c > z_pos:
            starts.append(c)
            z_pos = c
    return starts


def window_model(win):
    """[(start, end, seqs of the twin whose match starts in [start, end))] for every sub-block of a window."""
    seqs = lz4_sequences(lz4_twin_block(win))
    st = sub_blocks(seqs, len(win)) + [len(win)]
    out = []
    for a, b in zip(st[:-1], st[1:]):
        sel = seqs[(seqs[:, 0] >= a) & (seqs[:, 0] < b)] if len(seqs) else seqs
        out.append((a, b, sel))
    return out


def sub_block_literals(win, a, b, seqs):
    """The literal bytes of sub-block [a, b) with matches `seqs`."""
    keep = np.ones(b - a, bool)
    for s, _, ml in seqs:
        keep[s - a: s - a + ml] = False
    return np.asarray(win[a:b])[keep]


def huf_lengths(hist, limit=True):
    """Code length per symbol (dict) and the largest length, as zstd_entropy.cuh builds them: present symbols in
    ascending (count, symbol) order; two queues (leaves, internal nodes), the leaf taken on ties; depths from the tree;
    then, if the deepest leaf is below 11, clamp to 11, repay the Kraft excess by lengthening the first (rarest) leaf
    whose lengthening fits in what is left, else the rarest still short leaf, and hand back any overshoot by shortening
    11-bit codes, rarest first."""
    order = sorted((int(c), s) for s, c in enumerate(hist) if c)
    n = len(order)
    cnt = [c for c, _ in order] + [0] * (n - 1)
    par = [0] * (2 * n - 1)
    li, ii, ni = 0, n, n
    for _ in range(n - 1):
        pick = []
        for _ in range(2):
            if li < n and (ii >= ni or cnt[li] <= cnt[ii]):
                pick.append(li); li += 1
            else:
                pick.append(ii); ii += 1
        cnt[ni] = cnt[pick[0]] + cnt[pick[1]]; par[pick[0]] = par[pick[1]] = ni; ni += 1
    depth = [0] * (2 * n - 1)
    for v in range(ni - 2, -1, -1):
        depth[v] = depth[par[v]] + 1
    ln = depth[:n]
    maxl = max(ln)
    if limit and maxl > HUF_MAXBITS:
        ln = [min(x, HUF_MAXBITS) for x in ln]
        excess = sum(1 << (HUF_MAXBITS - x) for x in ln) - (1 << HUF_MAXBITS)
        while excess > 0:
            best = -1
            for i in range(n):
                if ln[i] < HUF_MAXBITS:
                    if best < 0:
                        best = i
                    if (1 << (HUF_MAXBITS - 1 - ln[i])) <= excess:
                        best = i
                        break
            if best < 0:
                break
            excess -= 1 << (HUF_MAXBITS - 1 - ln[best]); ln[best] += 1
        for i in range(n):
            if excess >= 0:
                break
            if ln[i] == HUF_MAXBITS:
                ln[i] -= 1; excess += 1
        maxl = HUF_MAXBITS
    return {s: ln[i] for i, (_, s) in enumerate(order)}, maxl


def kraft(lengths, maxbits):
    """Kraft sum in units of 2^-maxbits (complete code: exactly 1 << maxbits)."""
    return sum(1 << (maxbits - x) for x in lengths.values())
