"""The host pipeline behind LZ4MT_* / ZSTDCB_* (reader thread, submit on the calling thread, writer thread), driven
through Python callbacks with 1 MiB chunks so that one call spans several batches.  Both codecs, both directions.

Pinned here: what a failing callback does to a call (return code, an in-order prefix of the stream written, no write
after a failed one, the call returns), the callback return value -> library error mapping, that a context created after
a failed call on the same thread writes the whole stream again from pooled slots, and framed streams (LZ4 and zstd)
with frames larger than a decompress staging slot, or with more zstd blocks than its block table holds."""
import concurrent.futures
import ctypes
import queue
import struct
import threading

import numpy as np
import pytest

import _oracle as o
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu

CHUNK = 1 << 20
SMAX = 1 << 64
DEADLINE = 300                              # seconds: a call that has not returned by then hangs

# (mem, read_fail, canceled) of each codec (include/lz4-mt.h, include/zstd-mt.h)
ERR = {z.CODEC_LZ4: {"mem": 1, "read_fail": 2, "canceled": 9}, z.CODEC_ZSTD: {"mem": 1, "read_fail": 3, "canceled": 10}}
RV_TO_ERR = {-1: "read_fail", -2: "canceled", -3: "mem"}
API = {z.CODEC_LZ4: "LZ4MT", z.CODEC_ZSTD: "ZSTDCB"}


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


@pytest.fixture(scope="module")
def caller():
    """One host thread for every call of the module: a context created after a failed call runs on the same thread.  It
    is a daemon thread, so a call that hangs fails its test after DEADLINE and does not hold up the rest of the session."""
    jobs = queue.Queue()

    def work():
        for fn, fut in iter(jobs.get, None):
            try:
                fut.set_result(fn())
            except BaseException as e:
                fut.set_exception(e)

    threading.Thread(target=work, daemon=True).start()

    def call(fn):
        fut = concurrent.futures.Future()
        jobs.put((fn, fut))
        return fut.result(timeout=DEADLINE)
    yield call
    jobs.put(None)


def err(codec, rv):
    return SMAX - ERR[codec][RV_TO_ERR[rv]]


class Io:
    """fn_read serves `src`; fn_write records every frame.  fail_read / fail_write: index of the call that returns rv."""

    def __init__(self, src, fail_read=None, fail_write=None, rv=-1):
        self.src, self.pos, self.reads, self.writes = src, 0, 0, []
        self.fail_read, self.fail_write, self.rv = fail_read, fail_write, rv
        self.write_calls = 0
        self.rw = z.RdWr(z.RW_FN(self._rd), None, z.RW_FN(self._wr), None)

    def _rd(self, arg, b):
        i = self.reads; self.reads += 1
        if i == self.fail_read:
            return self.rv
        take = min(b.contents.size, self.src.size - self.pos)
        if take:
            ctypes.memmove(b.contents.buf, self.src[self.pos:].ctypes.data, take)
        self.pos += take; b.contents.size = take
        return 0

    def _wr(self, arg, b):
        i = self.write_calls; self.write_calls += 1
        if i == self.fail_write:
            return self.rv
        self.writes.append(ctypes.string_at(b.contents.buf, b.contents.size))
        return 0


def run(caller, codec, comp, io, level=1, threads=4):
    """One create / call / free on the caller's thread; returns the call's return code."""
    L = z.lib(); api = API[codec]

    def go():
        ctx = getattr(L, api + "_createCCtx")(threads, level if codec == z.CODEC_LZ4 else 3, CHUNK) if comp else \
            getattr(L, api + "_createDCtx")(threads, 0)
        assert ctx
        rc = getattr(L, api + ("_compressCCtx" if comp else "_decompressDCtx"))(ctx, ctypes.byref(io.rw))
        getattr(L, api + ("_freeCCtx" if comp else "_freeDCtx"))(ctx)
        return rc
    return caller(go)


def frames_of(framed):
    offs, sizes = z.scan_frames(framed)
    return [framed[int(a): int(a) + 12 + int(s)].tobytes() for a, s in zip(offs, sizes)]


def expected_frames(torch, codec, src):
    """Frames of `src` at CHUNK: the oracle's twin for LZ4, the device entry point for zstd (level 3)."""
    if codec == z.CODEC_LZ4:
        return frames_of(o.orc_encode_lz4(src, CHUNK))
    comp = z.ZstdDeviceCompressor(src.size, CHUNK)
    out, foff = comp.run(torch.from_numpy(src).cuda())
    torch.cuda.synchronize()
    return frames_of(out[: int(foff[-1].item())].cpu().numpy())


def assert_prefix(written, frames):
    assert written == frames[: len(written)], "frames written out of order or not those of the stream"


CODECS = [pytest.param(z.CODEC_LZ4, id="lz4"), pytest.param(z.CODEC_ZSTD, id="zstd")]


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("rv", [-1, -2, -3])
def test_compress_read_failure_in_third_batch(torch, caller, codec, rv):
    """8 chunks per batch: read 18 fails.  The reader stops there, the batches before may have been written, in order."""
    src = z.gen_stream(z.GEN_MIX, 40 * CHUNK + 77, CHUNK)
    io = Io(src, fail_read=18, rv=rv)
    assert run(caller, codec, True, io) == err(codec, rv)
    assert io.reads == 19
    assert len(io.writes) <= 16
    frames = expected_frames(torch, codec, src)
    assert_prefix(io.writes, frames)
    # a new context on the same thread, on the slots the failed call returned to the pool
    ok = Io(src)
    assert run(caller, codec, True, ok) == 0
    assert ok.writes == frames


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("rv", [-1, -2, -3])
def test_compress_write_failure_in_second_batch(torch, caller, codec, rv):
    src = z.gen_stream(z.GEN_MIX, 40 * CHUNK + 77, CHUNK)
    io = Io(src, fail_write=10, rv=rv)
    assert run(caller, codec, True, io) == err(codec, rv)
    assert io.write_calls == 11                                  # nothing is written after the failing frame
    frames = expected_frames(torch, codec, src)
    assert io.writes == frames[:10]
    ok = Io(src)
    assert run(caller, codec, True, ok) == 0
    assert ok.writes == frames


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("rv", [-1, -2, -3])
def test_framed_decompress_write_failure_in_second_batch(torch, caller, codec, rv):
    """Incompressible 1 MiB frames: about 31 fill a 32 MiB decompress batch, so frame 40 is in the second one."""
    n = 128 * CHUNK + 5
    src = z.gen_stream(z.GEN_RANDOM, n, CHUNK)
    rc, framed, _ = z.compress_mem(codec, src, threads=4, level=1 if codec == z.CODEC_LZ4 else 3, chunk=CHUNK)
    assert rc == 0
    io = Io(framed, fail_write=40, rv=rv)
    assert run(caller, codec, False, io) == err(codec, rv)
    assert io.write_calls == 41
    assert [len(w) for w in io.writes] == [CHUNK] * 40
    assert b"".join(io.writes) == src[: 40 * CHUNK].tobytes()
    ok = Io(framed)
    assert run(caller, codec, False, ok) == 0
    assert b"".join(ok.writes) == src.tobytes()


def test_lz4_frame_larger_than_the_decompress_slot(torch, caller):
    """A 40 MiB incompressible frame (a decompress slot holds 32 MiB of input), small frames, the large frame again and
    small frames: the reader grows the empty slot for a large first frame, and carries a large frame that arrives behind
    others over to the next batch."""
    big = z.gen_stream(z.GEN_RANDOM, 40 << 20, 40 << 20)
    small = z.gen_stream(z.GEN_MIX, 5 * CHUNK + 3, CHUNK)
    rc, f1, _ = z.compress_mem(z.CODEC_LZ4, big, threads=4, level=1, chunk=40 << 20)
    assert rc == 0
    rc, f2, _ = z.compress_mem(z.CODEC_LZ4, small, threads=4, level=1, chunk=CHUNK)
    assert rc == 0
    _, sizes = z.scan_frames(f1)
    assert len(sizes) == 1 and sizes[0] > 32 << 20
    framed = np.concatenate([f1, f2, f1, f2])
    io = Io(framed)
    assert run(caller, z.CODEC_LZ4, False, io) == 0
    assert [len(w) for w in io.writes] == ([40 << 20] + [CHUNK] * 5 + [3]) * 2
    assert b"".join(io.writes) == np.concatenate([big, small, big, small]).tobytes()


def zstd_raw_frame(content, block):
    """A framed zstd frame (12-byte header + payload) of raw blocks of `block` bytes, content size in the header."""
    parts = [struct.pack("<IBI", 0xFD2FB528, 0xA0, content.size)]                 # single segment, 4-byte content size
    for a in range(0, content.size, block):
        n = min(block, content.size - a)
        parts += [struct.pack("<I", (n << 3) | (a + n == content.size))[:3], content[a:a + n].tobytes()]
    payload = b"".join(parts)
    return np.frombuffer(struct.pack("<III", 0x184D2A50, 4, len(payload)) + payload, np.uint8)


def test_zstd_frames_larger_than_the_decompress_slot(torch, caller):
    """zstd frames that do not fit a decompress slot as it is: a 40 MiB frame of raw blocks (the slot holds 32 MiB of
    input), a frame of 33 000 raw blocks (the block table holds 32 768), and an 80 MiB compressed frame (the slot holds
    64 MiB of output), between small frames.  The reader grows the empty slot for each of them, first in its batch or
    carried over to the next one."""
    big = z.gen_stream(z.GEN_RANDOM, 40 << 20, 40 << 20)
    many = z.gen_stream(z.GEN_MIX, 33000 * 16, CHUNK)
    text = z.gen_stream(z.GEN_TEXT, 80 << 20, 80 << 20)
    small = z.gen_stream(z.GEN_MIX, 5 * CHUNK + 3, CHUNK)
    f_big, f_many = zstd_raw_frame(big, 128 << 10), zstd_raw_frame(many, 16)
    rc, f_text, _ = z.compress_mem(z.CODEC_ZSTD, text, threads=4, level=3, chunk=80 << 20)
    assert rc == 0
    rc, f_small, _ = z.compress_mem(z.CODEC_ZSTD, small, threads=4, level=3, chunk=CHUNK)
    assert rc == 0
    assert z.scan_frames(f_big)[1][0] > 32 << 20 and len(z.scan_frames(f_text)[1]) == 1
    framed = np.concatenate([f_big, f_small, f_many, f_big, f_text, f_small])
    io = Io(framed)
    assert run(caller, z.CODEC_ZSTD, False, io) == 0
    smalls = [CHUNK] * 5 + [3]
    assert [len(w) for w in io.writes] == [40 << 20] + smalls + [many.size, 40 << 20, 80 << 20] + smalls
    assert b"".join(io.writes) == np.concatenate([big, small, many, big, text, small]).tobytes()
