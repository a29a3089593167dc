"""The GPU LZ4 decoder on the edge corpus of _lz4corpus.py (frames written from dictated parses and accepted by liblz4):
every case in both layouts (two-pass path and frame-sequential fallback), all cases in one batch at every input
alignment, the callback API, XXH32 content checksums, LZ4F block checksums, and malformed
blocks aimed at each of the decoder's checks."""
import numpy as np
import pytest

import _lz4corpus as lc
import _oracle as o
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu
CASES = list(lc.CASES)
ST_BLOCK, ST_CONTENT_CHECKSUM = 5, 7


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def header(n):
    return np.frombuffer((0x184D2A50).to_bytes(4, "little") + (4).to_bytes(4, "little") + int(n).to_bytes(4, "little"), np.uint8)


def framed(frames, shifts=None):
    """Frames behind 12-byte headers, back to back; with shifts, pad bytes in front of each header put the LZ4F frame i
    (after its header) at input offset = shifts[i] mod 16 (the decoder takes any offsets)."""
    parts, offs, pos = [], [], 0
    for i, f in enumerate(frames):
        pad = (shifts[i] - (pos + 12)) % 16 if shifts else 0
        parts += [np.zeros(pad, np.uint8), header(f.size), f]
        offs.append(pos + pad); pos += pad + 12 + f.size
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8), offs


def device_decode(torch, frames, outs, shifts=None):
    """One zmt_lz4_decompress_device call: (decoder, output, status, sizes, needs_seq) per frame."""
    buf, offs = framed(frames, shifts)
    dec = z.Lz4DeviceDecompressor(offs, [f.size for f in frames], outs)
    out, st = dec.run(torch.from_numpy(buf).cuda())
    torch.cuda.synchronize()
    n = len(frames)
    a256 = lambda x: (x + 255) // 256 * 256
    ns = dec.work[2 * a256(4 * n): 2 * a256(4 * n) + 4 * n].view(torch.int32).cpu().numpy()       # workspace: stored | computed | needs_seq
    return dec, out[: max(dec.out_total, 1)].cpu().numpy(), st.cpu().numpy()[:n], dec.out_size.cpu().numpy()[:n], ns


def check(out, st, sz, srcs, bad=()):
    pos = 0
    for i, s in enumerate(srcs):
        if i not in bad:
            assert st[i] == 0, (i, z.ST_NAMES.get(int(st[i]), st[i]))
            assert sz[i] == s.size, i
            assert np.array_equal(out[pos: pos + s.size], s), i
        pos += s.size


@pytest.mark.parametrize("lay", lc.LAYOUTS)
@pytest.mark.parametrize("name", CASES)
def test_gpu_decodes_each_case_alone(gpu, name, lay):
    """(a) Every case as a batch of its own, in both layouts: status 0, the right sizes, the source bit for bit."""
    fr = lc.case(name, lay)
    _, out, st, sz, _ = device_decode(gpu, [f for f, _, _ in fr], [s.size for _, s, _ in fr])
    check(out, st, sz, [s for _, s, _ in fr])


def _all(bchk=False):
    items = [(n, lay, f, s) for lay in lc.LAYOUTS for n in CASES for f, s, _ in lc.case(n, lay, bchk)]
    return items, [i % 16 for i in range(len(items))]


@pytest.fixture(scope="module")
def batch(gpu):
    items, shifts = _all()
    res = device_decode(gpu, [f for _, _, f, _ in items], [s.size for *_, s in items], shifts)
    return items, shifts, res


def test_gpu_decodes_all_cases_in_one_batch_at_every_alignment(batch):
    """(b) All cases in one batch, frame i starting at input offset i mod 16: exactly the short frames of two or more
    blocks, and the frames with a zero-size block, take the frame-sequential pass (needs_seq), as the model says."""
    items, shifts, (dec, out, st, sz, ns) = batch
    check(out, st, sz, [s for *_, s in items])
    _, offs = framed([f for _, _, f, _ in items], shifts)
    starts = [(int(x) + 12) % 16 for x in offs]
    assert starts == [i % 16 for i in range(len(items))] and set(starts) == set(range(16))
    for i, (n, lay, f, s) in enumerate(items):
        tr = o.lz4f_trace(f, s.size)
        want = lc.expect_fallback(tr, (int(f[5]) >> 4) & 7)
        assert want == lc.expect_path_is_sequential(lay, tr), (n, lay)
        assert bool(ns[i]) == want, (i, n, lay)


@pytest.mark.parametrize("name", CASES)
def test_gpu_callback_api_decodes_each_case(gpu, name):
    """(d) LZ4MT_decompressDCtx on every case (both layouts), behind 12-byte headers and as a plain .lz4 stream."""
    for lay in lc.LAYOUTS:
        fr = lc.case(name, lay)
        src = np.concatenate([s for _, s, _ in fr])
        for stream in (framed([f for f, _, _ in fr])[0], np.concatenate([f for f, _, _ in fr])):
            rc, back, stt = z.decompress_mem(z.CODEC_LZ4, stream, src.size + 16, threads=4)
            assert rc == 0, z.lib().LZ4MT_getErrorString(rc)
            assert back.size == src.size and np.array_equal(back, src), (name, lay)


CHK_SIZES = list(range(41)) + [63, 64, 65, 511, 512, 513, 2047, 2048, 2049] + [(1 << 20) + r for r in range(32)]


def _chk_frame(n, i):
    if n == 0:
        spec = dict(blocks=[], cchk=True)
    elif n < 64:
        spec = dict(blocks=[[(n, 0, 0)]], cchk=True)
    else:
        spec = dict(blocks=[lc.close([(16, 8, 4), (200, 100, 30)] if n > 300 else [(16, 8, 4)], n)], bsid=7 if n > 65536 else 4, cchk=True)
    return lc.write_frame(spec, seed=i)[:2]


def test_gpu_content_checksum_tail_lengths(gpu):
    """(e) XXH32 content checksums over 0-40, 63-65, 511-513, 2047-2049 and 1 MiB + 0..31 bytes, with outputs starting at
    every residue mod 16 (the 16-byte-tile, 4-byte and byte load paths of the hash kernel); one flipped stored bit fails
    exactly the damaged frames with ZMT_ST_CONTENT_CHECKSUM and leaves the others intact."""
    fs = [_chk_frame(n, i) for i, n in enumerate(CHK_SIZES)]
    frames, srcs = [f for f, _ in fs], [s for _, s in fs]
    starts = np.cumsum([0] + [s.size for s in srcs])[:-1]
    assert set(int(x) % 16 for x in starts) == set(range(16))
    _, out, st, sz, _ = device_decode(gpu, frames, [s.size for s in srcs])
    check(out, st, sz, srcs)
    for parity in (0, 1):
        bad = [f.copy() for f in frames]
        for i in range(parity, len(bad), 2):
            bad[i][bad[i].size - 4 + (i // 8) % 4] ^= np.uint8(1 << (i % 8))
        _, out, st, sz, _ = device_decode(gpu, bad, [s.size for s in srcs])
        assert list(st) == [ST_CONTENT_CHECKSUM if i % 2 == parity else 0 for i in range(len(frames))]
        check(out, st, sz, srcs, bad={i for i in range(len(frames)) if i % 2 == parity})


def _damage(frame, src, kind, k):
    """A copy of the frame with its k-th checksummed block damaged: `sum` flips a bit of the stored block checksum,
    `data` flips a literal byte of the block (or any byte of a stored block) and leaves the checksum as it was."""
    tr = o.lz4f_trace(frame, src.size)
    cand = [b for b in range(len(tr.blk)) if tr.blk[b, o.L4B["bsize"]] > 0]
    b = cand[k % len(cand)]
    foff, bs = int(tr.blk[b, o.L4B["foff"]]), int(tr.blk[b, o.L4B["bsize"]])
    f = frame.copy()
    if kind == "sum":
        f[foff + bs + k % 4] ^= np.uint8(1 << (k % 8))
    elif tr.blk[b, o.L4B["stored"]]:
        f[foff + bs // 2] ^= np.uint8(0x40)
    else:
        sq = tr.block_seqs(b)
        r = sq[np.flatnonzero(sq[:, o.L4S["ll"]] > 0)[0]]
        f[int(r[o.L4S["tokpos"]]) + 1 + int(r[o.L4S["llext"]])] ^= np.uint8(0x40)
    rc, _, _ = o.lz4f_decode(f, src.size)
    assert rc == -5                                          # ORC_ERR_BLOCK: the oracle rejects it too
    return f


@pytest.mark.parametrize("lay", lc.LAYOUTS)
def test_gpu_block_checksums(gpu, lay):
    """(f) The corpus written with FLG.BC decodes; a flipped block-checksum bit, and separately a flipped payload byte
    under an intact checksum, fail exactly the damaged frames with ZMT_ST_BLOCK while the rest of the batch decodes; the
    callback API refuses the damaged plain stream, as liblz4 does."""
    items = [(f, s) for n in CASES for f, s, _ in lc.case(n, lay, True)]
    frames, srcs = [f for f, _ in items], [s for _, s in items]
    outs = [s.size for s in srcs]
    assert all(f[4] & 0x10 for f in frames)
    _, out, st, sz, _ = device_decode(gpu, frames, outs)
    check(out, st, sz, srcs)
    hit = [i for i, s in enumerate(srcs) if s.size > 0]
    for kind in ("sum", "data"):
        for parity in (0, 1):
            bad = set(hit[parity::2])
            dam = [_damage(f, s, kind, i) if i in bad else f for i, (f, s) in enumerate(items)]
            _, out, st, sz, _ = device_decode(gpu, dam, outs)
            assert [int(x) for x in st] == [ST_BLOCK if i in bad else 0 for i in range(len(frames))], (kind, parity)
            check(out, st, sz, srcs, bad=bad)
        i = hit[0]
        plain = _damage(frames[i], srcs[i], kind, 0)
        msg, _ = lc.liblz4_frame(plain, srcs[i].size)
        assert isinstance(msg, str) and "Checksum" in msg, msg
        rc, _, _ = z.decompress_mem(z.CODEC_LZ4, plain, srcs[i].size + 16, threads=4)
        assert z.lib().LZ4MT_isError(rc)


def _malformed():
    """(name, frame, output size) of one block aimed at each check of the decoder."""
    rng = np.random.default_rng(77)
    raw = lambda n: rng.integers(0, 256, n, dtype=np.uint8)

    def frame(blocks, bsid=4, linked=False):
        hd = bytes([0x40 | (0 if linked else 0x20), bsid << 4])
        out = bytearray((0x184D2204).to_bytes(4, "little")) + hd + bytes([(o.xxh32(np.frombuffer(hd, np.uint8)) >> 8) & 0xFF])
        for hdr, data in blocks:
            out += int(hdr).to_bytes(4, "little") + data
        return np.frombuffer(bytes(out + bytes(4)), np.uint8).copy()

    src = raw(70000)
    blk = lambda rows, p=0: lc.write_block(rows, src, p)
    b = blk([(20, 0, 10), (16, 0, 0)]); yield "offset 0", frame([(len(b), b)]), 46
    b = blk([(20, 21, 10), (16, 0, 0)]); yield "offset op + hist + 1, independent", frame([(len(b), b)]), 46
    b0 = blk([(100, 0, 0)]); b1 = blk([(0, 101, 10), (16, 0, 0)], 100)
    yield "offset op + hist + 1, linked", frame([(len(b0), b0), (len(b1), b1)], linked=True), 126
    b = blk([(20, 1, 65600), (16, 0, 0)]); yield "match past the output room", frame([(len(b), b)]), 65636
    b = blk([(50, 0, 0)])[:-10]; yield "literal run past the block end", frame([(len(b), b)]), 50
    yield "block size > blockMaxSize", frame([(65537 | 0x80000000, src[:65537].tobytes())]), 65537


@pytest.mark.parametrize("k", range(6))
def test_gpu_malformed_blocks(gpu, k):
    """(g) Malformed blocks, one per check of the decoder: the oracle rejects each, and liblz4 every one but offset 0 (the
    format calls a zero offset invalid; liblz4 1.9.4 does not test for it and copies from the output position itself); on
    the GPU the frame fails with ZMT_ST_BLOCK and its neighbours decode intact."""
    name, bad, n = list(_malformed())[k]
    msg, _ = lc.liblz4_frame(bad, n)
    assert isinstance(msg, str) or name == "offset 0", name
    rc, _, _ = o.lz4f_decode(bad, n)
    assert rc in (-5, -6), (name, rc)
    (f0, s0, _), (f1, s1, _) = lc.case("ends")[0], lc.case("lengths")[0]
    _, out, st, sz, _ = device_decode(gpu, [f0, bad, f1], [s0.size, n, s1.size])
    assert int(st[1]) == ST_BLOCK, (name, z.ST_NAMES.get(int(st[1])))
    assert st[0] == 0 and st[2] == 0
    assert np.array_equal(out[: s0.size], s0) and np.array_equal(out[s0.size + n: s0.size + n + s1.size], s1)
