"""The LZ4 level-1 compressor (lz4_blocks_pipe_kernel) and the zstd level-3 encoder (zstd_blocks_kernel) on the edge
corpus of tests/_pipecorpus.py (pytest -m gpu).  LZ4: the stream is byte for byte the CPU twin's (orc_encode_lz4) and
decodes through the oracle and, when oracle/_ref exists, the reference.  zstd: test_gpu_zstd_encoder.check compares
the parse with the twin sub-block by sub-block and round-trips every frame.  The batch cases stage blocks whose size
is not a multiple of 16 and blocks at every address mod 16 (the byte-copy path of lz_stage), the persistent-loop case
makes each CTA's second block follow an edge block, and the host pipeline runs once per codec on an input whose size
is not a multiple of 16."""
import numpy as np
import pytest

import _oracle as o
import _pipecorpus as pc
import test_gpu_zstd_encoder as tz
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu
BUILT = {b.__name__: b() for b in pc.BUILDERS}
CHUNK = 1 << 20
BATCH_WIN = 24 << 10


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def case_parts(name):
    src, chunk, marks, _ = BUILT[name]
    return pc.parts(src, chunk, marks), chunk


def lz4_device(torch, d_in, n, chunk, sizes=None):
    """zmt_lz4_compress_level_device at level 1 on d_in (explicit chunk sizes: chunk c at d_in + c * chunk)."""
    L = z.lib()
    nch = len(sizes) if sizes is not None else L.zmt_chunk_count(n, chunk)
    d_cb = torch.from_numpy(np.asarray(sizes, np.int32)).cuda() if sizes is not None else None
    work = torch.empty(L.zmt_lz4c_level_workspace_bytes(nch, chunk, 1), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_lz4c_out_bound(nch, chunk), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(nch + 1, dtype=torch.int64, device="cuda")
    rc = L.zmt_lz4_compress_level_device(d_in.data_ptr(), n, chunk, d_cb.data_ptr() if d_cb is not None else None, nch, 1,
                                         work.data_ptr(), out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy()


def lz4_expect(parts, chunk):
    return np.concatenate([o.orc_encode_lz4(p, chunk) for p in parts])


def check_lz4_decodes(framed, parts):
    want = np.concatenate(parts)
    rc, back = o.orc_decode(o.CODEC_LZ4, framed, want.size)
    assert rc == 0 and np.array_equal(back, want)
    if o.have_ref():
        rc, back, _ = o.ref_decompress(o.CODEC_LZ4, framed, want.size)
        assert rc == 0 and np.array_equal(back, want)


def padded(parts, stride):
    """The parts at a stride of `stride` bytes, and their sizes (explicit chunk sizes)."""
    src = np.zeros(len(parts) * stride, np.uint8)
    for c, p in enumerate(parts):
        src[c * stride: c * stride + p.size] = p
    return src, [int(p.size) for p in parts]


# ------------------------------------------------------------------------------------------------- the corpus
@pytest.mark.parametrize("name", list(BUILT))
def test_lz4_corpus_case(torch, name):
    parts, chunk = case_parts(name)
    if chunk is None:                                            # explicit sizes: one chunk per part
        src, sizes = padded(parts, 64)
        framed = lz4_device(torch, torch.from_numpy(src).cuda(), src.size, 64, sizes)
        expect = lz4_expect(parts, 64)
    else:
        src = np.concatenate(parts)
        framed = lz4_device(torch, torch.from_numpy(src).cuda(), src.size, chunk)
        expect = o.orc_encode_lz4(src, chunk)
    assert framed.size == expect.size and np.array_equal(framed, expect), "GPU stream differs from the oracle twin"
    check_lz4_decodes(framed, parts)


@pytest.mark.parametrize("name", list(BUILT))
def test_zstd_corpus_case(torch, name):
    parts, chunk = case_parts(name)
    if chunk is None:
        src, sizes = padded(parts, 64)
        tz.check(torch, src, 64, sizes)
    else:
        tz.check(torch, np.concatenate(parts), chunk)


# ------------------------------------------------------------------------------------------------- staging
def batch_parts():
    """Every case's content cut into chunks of at most 24 KiB whose sizes are = 1..15 mod 16 in turn (each loses its
    last 1..15 bytes), so that every chunk's last block ends off a 16-byte boundary: the bulk copy stages its whole
    16-byte words and the byte loop of lz_stage the 1..15 bytes after them.  The chunks themselves start at multiples
    of 24 KiB; starts off a 16-byte boundary are the address tests' part."""
    out = []
    for name in BUILT:
        for p in case_parts(name)[0]:
            for a in range(0, p.size, BATCH_WIN):
                q = p[a: a + BATCH_WIN]
                r = len(out) % 15 + 1
                k = q.size - (q.size - r) % 16
                if k > 0:
                    out.append(q[:k])
    return out


def test_lz4_batch_sizes_off_16(torch):
    parts = batch_parts()
    assert {p.size % 16 for p in parts} >= set(range(1, 16))
    src, sizes = padded(parts, BATCH_WIN)
    framed = lz4_device(torch, torch.from_numpy(src).cuda(), src.size, BATCH_WIN, sizes)
    assert np.array_equal(framed, lz4_expect(parts, BATCH_WIN))
    check_lz4_decodes(framed, parts)


def test_zstd_batch_sizes_off_16(torch):
    parts = batch_parts()
    src, sizes = padded(parts, BATCH_WIN)
    tz.check(torch, src, BATCH_WIN, sizes)


STRIDE = 3 * pc.LB                       # the longest chunk of any case


def corpus_layout():
    """Every chunk of every case at a stride of STRIDE bytes, with its size: each case keeps its own block and tile
    layout (a chunk's blocks are cut from its start)."""
    parts = [p for name in BUILT for p in case_parts(name)[0]]
    assert max(p.size for p in parts) <= STRIDE
    src, sizes = padded(parts, STRIDE)
    return parts, src, sizes


def zstd_device(torch, d_in, chunk, sizes):
    """zmt_zstd_compress_device on d_in with explicit chunk sizes (chunk c at d_in + c * chunk)."""
    L = z.lib()
    nch = len(sizes)
    d_cb = torch.from_numpy(np.asarray(sizes, np.int32)).cuda()
    work = torch.empty(L.zmt_zstdc_workspace_bytes(nch, chunk), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_zstdc_out_bound(nch, chunk), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(nch + 1, dtype=torch.int64, device="cuda")
    rc = L.zmt_zstd_compress_device(d_in.data_ptr(), d_in.numel(), chunk, d_cb.data_ptr(), nch, work.data_ptr(),
                                    out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy()


def at_offsets(torch, src):
    """The same bytes on the device starting at every address mod 16 (one buffer, rewritten per offset)."""
    buf = torch.zeros(src.size + 16, dtype=torch.uint8, device="cuda")
    d_src = torch.from_numpy(src).cuda()
    for a in range(16):
        buf[a: a + src.size] = d_src
        d_in = buf[a: a + src.size]
        assert d_in.data_ptr() % 16 == a
        yield a, d_in


def test_lz4_input_at_every_address_mod_16(torch):
    """Every case's chunks, in their own layout, from a device pointer at each address mod 16: off 16 every block is
    staged byte by byte (no bulk copy), and the stream is the twin's every time."""
    parts, src, sizes = corpus_layout()
    expect = lz4_expect(parts, STRIDE)
    for a, d_in in at_offsets(torch, src):
        framed = lz4_device(torch, d_in, src.size, STRIDE, sizes)
        assert np.array_equal(framed, expect), ("stream differs at input address mod 16", a)
    check_lz4_decodes(expect, parts)


def test_zstd_input_at_every_address_mod_16(torch):
    """As above for the zstd encoder: the aligned run is checked against the twin, every other address must write the
    same frames."""
    parts, src, sizes = corpus_layout()
    tz.check(torch, src, STRIDE, sizes)
    ref = tz.gpu_compress(torch, src, STRIDE, sizes)
    for a, d_in in at_offsets(torch, src):
        assert np.array_equal(zstd_device(torch, d_in, STRIDE, sizes), ref), ("stream differs at input address mod 16", a)


# ------------------------------------------------------------------------------------------------- persistent loop
def corpus_windows():
    wins = []
    for name in BUILT:
        for p in case_parts(name)[0]:
            wins += [p[a: a + pc.LB] for a in range(0, p.size, pc.LB) if p[a: a + pc.LB].size >= 16]
    return wins


def two_per_cta(grid, wins):
    """2 * grid one-block chunks: block i and block i + grid (the next one CTA i encodes) are different corpus windows,
    each the edge window of the other's state."""
    src = np.zeros(2 * grid * pc.LB, np.uint8)
    sizes = []
    for c in range(2 * grid):
        w = wins[(c + c // grid) % len(wins)]
        src[c * pc.LB: c * pc.LB + w.size] = w
        sizes.append(int(w.size))
    return src, sizes


def test_lz4_each_cta_encodes_two_edge_blocks(torch, capsys):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    grid = 16 * sm
    wins = corpus_windows()
    src, sizes = two_per_cta(grid, wins)
    framed = lz4_device(torch, torch.from_numpy(src).cuda(), src.size, pc.LB, sizes)
    parts = [src[c * pc.LB: c * pc.LB + s] for c, s in enumerate(sizes)]
    assert np.array_equal(framed, lz4_expect(parts, pc.LB))
    with capsys.disabled():
        print("\n[persistent] lz4: grid %d, %d blocks, %d MB" % (grid, len(sizes), src.size >> 20))


def test_zstd_each_cta_encodes_two_edge_blocks(torch, capsys):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    grid = min(8 * sm, 132 * 8)
    wins = corpus_windows()
    src, sizes = two_per_cta(grid, wins)
    tz.check(torch, src, pc.LB, sizes)
    with capsys.disabled():
        print("\n[persistent] zstd: grid %d, %d blocks, %d MB" % (grid, len(sizes), src.size >> 20))


# ------------------------------------------------------------------------------------------------- host pipeline
@pytest.mark.parametrize("codec", [z.CODEC_LZ4, z.CODEC_ZSTD])
def test_host_pipeline_size_off_16(torch, codec):
    """{LZ4MT,ZSTDCB}_compressCCtx on the corpus with an input size of 7 mod 16 writes what the device path writes."""
    _, src, _ = corpus_layout()                  # chunks of STRIDE bytes: each case keeps its layout
    src = src[: src.size - (src.size - 7) % 16]
    rc, framed, _ = z.compress_mem(codec, src, threads=4, level=1 if codec == z.CODEC_LZ4 else 3, chunk=STRIDE)
    assert rc == 0
    if codec == z.CODEC_LZ4:
        dev = lz4_device(torch, torch.from_numpy(src).cuda(), src.size, STRIDE)
        assert np.array_equal(dev, o.orc_encode_lz4(src, STRIDE))
    else:
        comp = z.ZstdDeviceCompressor(int(src.size), STRIDE)
        out, foff = comp.run(torch.from_numpy(src).cuda())
        torch.cuda.synchronize()
        dev = out[: int(foff[-1].item())].cpu().numpy()
    assert np.array_equal(framed, dev)
    rc, back = o.orc_decode(codec, framed, src.size)
    assert rc == 0 and np.array_equal(back, src)
