"""The size contract of the device decoders, the frame index and range reads (pytest -m gpu): each call writes nothing
past the bytes its *_workspace_bytes function asks for, and what the workspace held before the call does not change
its results.  Each call runs once on an exactly sized, zeroed workspace and once on a workspace with a guard tail, all of
it filled with 0xA5; the tail must come back untouched and the outputs, sizes and statuses equal."""
import ctypes
import json
import os

import numpy as np
import pytest

import _lz4corpus as lc
import _zcorpus as zc
import zstdmt_b200 as z
from test_gpu_frame_index import framed, host_lz4, host_zstd

pytestmark = pytest.mark.gpu
GUARD = 1 << 16
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def golden(name):
    case = next(c for c in json.load(open(os.path.join(GOLD, "manifest.json")))["cases"] if c["file"] == name)
    return np.fromfile(os.path.join(GOLD, name), dtype=np.uint8), z.gen_stream(case["kind"], case["n"], case["chunk"], first=case["first"])


def twice(torch, sizes, call, init=()):
    """call(*works) enqueues one entry point on workspaces of `sizes` bytes (the first len(init) start with those bytes)
    and returns the tensors it wrote.  Exact and zeroed first, then 0xA5 with a guard tail; returns the second results."""
    def works(fill, extra):
        ws = [torch.full((n + extra,), fill, dtype=torch.uint8, device="cuda") for n in sizes]
        for w, t in zip(ws, init):
            w[: t.numel()] = t
        return ws
    assert all(n > 0 for n in sizes)
    first = [t.clone() for t in call(*works(0, 0))]
    torch.cuda.synchronize()
    ws = works(0xA5, GUARD)
    second = call(*ws)
    torch.cuda.synchronize()
    for w, n in zip(ws, sizes):
        assert bool((w[n:] == 0xA5).all()), "the call wrote past its workspace"
    for a, b in zip(first, second):
        assert torch.equal(a, b), "the results depend on what the workspace held"
    return second


def cu(torch, a, dtype=None):
    a = np.ascontiguousarray(a if dtype is None else np.asarray(a).astype(dtype))
    return torch.from_numpy(a.view(np.uint8) if a.size else np.zeros(8, np.uint8)).cuda()


def stream(torch):
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------ decoders
def lz4_decode(torch, fb, srcs):
    L = z.lib()
    offs, sizes, out_off, slots = host_lz4(fb)
    n = len(offs)
    d_in, d_off, d_cs, d_oo = cu(torch, fb), cu(torch, offs, np.int64), cu(torch, sizes, np.int32), cu(torch, out_off, np.int64)

    def call(work):
        out = torch.zeros(max(int(out_off[-1]), 1), dtype=torch.uint8, device="cuda")
        osz, st = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
        rc = L.zmt_lz4_decompress_device(d_in.data_ptr(), fb.size, d_off.data_ptr(), d_cs.data_ptr(), n, slots, out.data_ptr(), d_oo.data_ptr(),
                                         osz.data_ptr(), st.data_ptr(), work.data_ptr(), stream(torch))
        assert rc == 0, z.ST_NAMES.get(rc, rc)
        return [out, osz, st]
    out, osz, st = twice(torch, [L.zmt_lz4d_workspace_bytes(n, slots, fb.size)], call)
    assert not st.cpu().numpy().any()
    for i, s in enumerate(srcs):
        assert int(osz[i]) == s.size and np.array_equal(out[int(out_off[i]): int(out_off[i]) + s.size].cpu().numpy(), s), i


def zstd_decode(torch, fb, srcs):
    L = z.lib()
    h = host_zstd(fb)
    n, nblk = len(h["frame_off"]), len(h["blocks"]) // L.zmt_zstd_blk_desc_bytes()
    d_in, d_blk, d_first = cu(torch, fb), cu(torch, h["blocks"]), cu(torch, h["first"])
    d_exp, d_seq, d_oo = cu(torch, h["expect"]), cu(torch, h["flags"]), cu(torch, h["out_off"])

    def call(work):
        out = torch.zeros(max(int(h["out_off"][-1]), 1), dtype=torch.uint8, device="cuda")
        osz, st = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
        rc = L.zmt_zstd_decompress_device(d_in.data_ptr(), d_blk.data_ptr(), nblk, d_first.data_ptr(), d_exp.data_ptr(), d_seq.data_ptr(), n,
                                          out.data_ptr(), d_oo.data_ptr(), osz.data_ptr(), st.data_ptr(), work.data_ptr(), stream(torch))
        assert rc == 0, z.ST_NAMES.get(rc, rc)
        return [out, osz, st]
    out, osz, st = twice(torch, [L.zmt_zstdd_workspace_bytes(n, nblk, h["scratch"])], call)
    assert not st.cpu().numpy().any()
    oo = h["out_off"].astype(np.int64)
    for i, s in enumerate(srcs):
        assert int(osz[i]) == s.size and np.array_equal(out[oo[i]: oo[i] + s.size].cpu().numpy(), s), i


def test_lz4_independent_blocks(torch):
    fb, src = golden("lz4_l1_k2_196625.bin")
    lz4_decode(torch, fb, [src[:131072], src[131072:]])


@pytest.mark.parametrize("bchk", [False, True], ids=["linked", "linked_bchk"])
def test_lz4_linked_blocks_and_block_checksums(torch, bchk):
    items = [(f, s) for name in ("linked", "lengths") for f, s, _ in lc.case(name, "full", bchk)]
    lz4_decode(torch, framed([f for f, _ in items]), [s for _, s in items])


def test_zstd_self_contained_frames(torch):
    fb, src = golden("zstd_l3_k2_196613.bin")
    zstd_decode(torch, fb, [src[i: i + 65536] for i in range(0, src.size, 65536)])


def test_zstd_dependent_blocks(torch):
    cases = [zc.case(name) for name in ("reps", "tables")]
    zstd_decode(torch, framed([f for _, f in cases]), [s for s, _ in cases])


def test_lz4_segments(torch):
    """One linked frame as segments of about a third of it, each after the first reading the history before it."""
    L = z.lib()
    fr, src, _ = lc.case("linked")[0]
    flg, bd, H = int(fr[4]), int(fr[5]), 65536
    seg = torch.zeros(ctypes.sizeof(z.Lz4Segment), dtype=torch.uint8, device="cuda")
    prev, hist, got, last = 0, np.zeros(0, np.uint8), [], 0
    while not last:
        k = len(got)
        rc, end, room, last = z.lz4f_segment(fr[prev:], (7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)) if k == 0 else 0, flg, bd,
                                             fr.size // 3, 1 << 62)
        assert rc == 0
        d_in = torch.zeros(12 + end + 256, dtype=torch.uint8, device="cuda")
        d_in[12:12 + end] = cu(torch, fr[prev:prev + end])
        rec = z.Lz4Segment.from_buffer_copy(bytes(seg.cpu().numpy()))
        rec.history, rec.flags = hist.size, (z.SEG_FIRST if k == 0 else 0) | (z.SEG_LAST if last else 0)
        rec_t = torch.frombuffer(bytearray(bytes(rec)), dtype=torch.uint8).cuda()
        foff, fcs = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.tensor([end], dtype=torch.int32, device="cuda")
        ooff = torch.tensor([H, H + room], dtype=torch.int64, device="cuda")
        nslots = max(1, (room + 65535) // 65536)

        def call(work):
            out = torch.zeros(H + room + 256, dtype=torch.uint8, device="cuda")
            out[H - hist.size:H] = cu(torch, hist)[: hist.size]
            s, osz, st = rec_t.clone(), torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
            rc = L.zmt_lz4_decompress_segments_device(d_in.data_ptr(), d_in.numel(), foff.data_ptr(), fcs.data_ptr(), 1, nslots, out.data_ptr(),
                                                      ooff.data_ptr(), osz.data_ptr(), st.data_ptr(), s.data_ptr(), work.data_ptr(), stream(torch))
            assert rc == 0, z.ST_NAMES.get(rc, rc)
            return [out, osz, st, s]
        out, osz, st, seg = twice(torch, [L.zmt_lz4d_workspace_bytes(1, nslots, d_in.numel())], call)
        assert int(st.item()) == 0
        part = out[H:H + int(osz.item())].cpu().numpy()
        got.append(part)
        hist = np.concatenate([hist, part])[-H:]
        prev += end
    assert len(got) >= 2 and prev == fr.size and np.array_equal(np.concatenate(got), src)


def test_zstd_segments(torch):
    """A frame with dependent blocks as segments of about a third of it: later ones carry table sources and read the history."""
    L = z.lib()
    src, fr = zc.case("reps")
    seg = torch.zeros(ctypes.sizeof(z.ZstdSegment), dtype=torch.uint8, device="cuda")
    w, prev, hist, got, last = z.ZstdWalk(), 0, np.zeros(0, np.uint8), [], 0
    while not last:
        k = len(got)
        carry = b"".join(fr[o:o + n].tobytes() for o, n in z.zstd_segment_sources(w))
        rc, end, room, flags, last, blk, scr = z.zstd_segment(fr[prev:], w, fr.size // 3, 1 << 62, base_off=len(carry))
        assert rc == 0
        nblk = blk.size // L.zmt_zstd_blk_desc_bytes()
        d_in = cu(torch, np.frombuffer(carry + fr[prev:prev + end].tobytes() + bytes(256), np.uint8))
        d_blk = cu(torch, blk)
        first = torch.tensor([0, nblk], dtype=torch.int32, device="cuda")
        expect = torch.tensor([-1 if k or flags & 4 else w.content_size], dtype=torch.int64, device="cuda")
        fseq = torch.tensor([flags], dtype=torch.int32, device="cuda")
        Hn = hist.size
        ooff = torch.tensor([Hn, Hn + room], dtype=torch.int64, device="cuda")
        rec = z.ZstdSegment.from_buffer_copy(bytes(seg.cpu().numpy()))
        rec.history, rec.flags = Hn, (z.SEG_FIRST if k == 0 else 0) | (z.SEG_LAST if last else 0)
        rec_t = torch.frombuffer(bytearray(bytes(rec)), dtype=torch.uint8).cuda()

        def call(work):
            out = torch.zeros(Hn + room + 256, dtype=torch.uint8, device="cuda")
            out[:Hn] = cu(torch, hist)[:Hn]
            s, osz, st = rec_t.clone(), torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
            rc = L.zmt_zstd_decompress_segments_device(d_in.data_ptr(), d_blk.data_ptr(), nblk, first.data_ptr(), expect.data_ptr(), fseq.data_ptr(), 1,
                                                       out.data_ptr(), ooff.data_ptr(), osz.data_ptr(), st.data_ptr(), s.data_ptr(), work.data_ptr(),
                                                       stream(torch))
            assert rc == 0, z.ST_NAMES.get(rc, rc)
            return [out, osz, st, s]
        out, osz, st, seg = twice(torch, [L.zmt_zstdd_workspace_bytes(1, nblk, scr)], call)
        assert int(st.item()) == 0
        part = out[Hn:Hn + int(osz.item())].cpu().numpy()
        got.append(part)
        hist = np.concatenate([hist, part])[-w.window:] if w.window else hist[:0]
        prev += end
    assert len(got) >= 2 and prev == fr.size and np.array_equal(np.concatenate(got), src)


# ------------------------------------------------------------------ frame index
def index(torch, fb, codec, plain, max_frames):
    L = z.lib()
    d = cu(torch, fb)
    m = max_frames

    def call(work):
        e = lambda k, dt: torch.zeros(max(k, 1), dtype=dt, device="cuda")
        t = [e(m, torch.int64), e(m, torch.int32), e(m + 1, torch.int64), e(40, torch.uint8)]
        if codec == "lz4":
            fn = L.zmt_lz4_index_plain_device if plain else L.zmt_lz4_index_device
            rc = fn(d.data_ptr(), fb.size, m, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), work.data_ptr(), stream(torch))
        else:
            t += [e(m + 1, torch.int32), e(m + 1, torch.int64), e(m, torch.int64), e(m, torch.int32)]
            fn = L.zmt_zstd_index_plain_device if plain else L.zmt_zstd_index_device
            rc = fn(d.data_ptr(), fb.size, m, t[0].data_ptr(), t[1].data_ptr(), *[x.data_ptr() for x in t[4:]], t[2].data_ptr(), t[3].data_ptr(),
                    work.data_ptr(), stream(torch))
        assert rc == 0, z.ST_NAMES.get(rc, rc)
        return t
    t = twice(torch, [L.zmt_index_workspace_bytes(m)], call)
    return z.FrameIndex.from_buffer_copy(t[3].cpu().numpy().tobytes())


@pytest.mark.parametrize("plain", [False, True], ids=["container", "plain"])
@pytest.mark.parametrize("name", ["lz4_l1_k3_2147.bin", "zstd_l3_k2_196613.bin"])
def test_index(torch, name, plain):
    fb, _ = golden(name)
    offs, sizes = z.scan_frames(fb)
    if plain:
        fb = np.concatenate([fb[int(o) + 12: int(o) + 12 + int(s)] for o, s in zip(offs, sizes)])
    codec, n = name[:name.index("_")], len(offs)
    info = index(torch, fb, codec, plain, n)
    assert (info.status, info.nframes) == (0, n)
    info = index(torch, fb, codec, plain, n - 1)                  # max_frames below the true count
    assert (info.status, info.nframes) == (6, n)                  # ZMT_ST_DST_SMALL


# ------------------------------------------------------------------ range reads
@pytest.mark.parametrize("name", ["lz4_l1_k3_2147.bin", "zstd_l3_k2_196613.bin"])
def test_range_reads(torch, name):
    L = z.lib()
    fb, src = golden(name)
    zstd = name.startswith("zstd")
    d = cu(torch, fb)
    info, t = z._device_index(d, None, torch.cuda.current_stream(), zstd=zstd)
    n, p = info.nframes, (lambda k: t[k].data_ptr())

    def content(work):
        off, d_info = torch.zeros(n + 1, dtype=torch.int64, device="cuda"), torch.zeros(40, dtype=torch.uint8, device="cuda")
        if zstd:
            rc = L.zmt_zstd_content_offsets_device(n, p("frame_off"), p("frame_csize"), p("expect"), off.data_ptr(), d_info.data_ptr(), work.data_ptr(),
                                                   stream(torch))
        else:
            rc = L.zmt_lz4_content_offsets_device(d.data_ptr(), n, p("frame_off"), p("frame_csize"), off.data_ptr(), d_info.data_ptr(), work.data_ptr(),
                                                  stream(torch))
        assert rc == 0, z.ST_NAMES.get(rc, rc)
        return [off, d_info]
    content_off, _ = twice(torch, [L.zmt_range_workspace_bytes(n, 0)], content)
    assert int(content_off[n]) == src.size

    rng = np.random.default_rng(7)
    starts = rng.integers(0, src.size, 40)
    ranges = np.stack([starts, np.minimum(rng.integers(0, 3000, 40), src.size - starts)], 1).astype(np.int64)
    d_ranges, m = cu(torch, ranges), len(ranges)
    wb = L.zmt_range_workspace_bytes(n, m)
    plan_work = []

    def plan(work):
        dst_off, d_plan = torch.zeros(m + 1, dtype=torch.int64, device="cuda"), torch.zeros(ctypes.sizeof(z.RangePlan), dtype=torch.uint8, device="cuda")
        if zstd:
            rc = L.zmt_zstd_range_plan_device(n, p("frame_csize"), p("first_blk"), p("frame_scratch"), content_off.data_ptr(), d_ranges.data_ptr(), m,
                                              dst_off.data_ptr(), d_plan.data_ptr(), work.data_ptr(), stream(torch))
        else:
            rc = L.zmt_lz4_range_plan_device(n, p("frame_csize"), content_off.data_ptr(), d_ranges.data_ptr(), m, dst_off.data_ptr(), d_plan.data_ptr(),
                                             work.data_ptr(), stream(torch))
        assert rc == 0, z.ST_NAMES.get(rc, rc)
        plan_work[:] = [work]
        return [dst_off, d_plan]
    dst_off, d_plan = twice(torch, [wb], plan)
    pl = z.RangePlan.from_buffer_copy(d_plan.cpu().numpy().tobytes())
    assert pl.status == 0 and pl.nsel > 0
    state = plan_work[0][:wb].clone()                             # the plan's tables, which the read call reads

    def read(work, read_work):
        out = torch.zeros(max(pl.dst_bytes, 1), dtype=torch.uint8, device="cuda")
        st, scratch = torch.zeros(m, dtype=torch.int32, device="cuda"), torch.zeros(max(pl.scratch_bytes, 1), dtype=torch.uint8, device="cuda")
        if zstd:
            rc = L.zmt_zstd_range_read_device(d.data_ptr(), p("frame_off"), p("frame_csize"), p("expect"), p("frame_seq"), ctypes.byref(pl), out.data_ptr(),
                                              dst_off.data_ptr(), st.data_ptr(), scratch.data_ptr(), read_work.data_ptr(), work.data_ptr(), stream(torch))
        else:
            rc = L.zmt_lz4_range_read_device(d.data_ptr(), p("frame_off"), p("frame_csize"), ctypes.byref(pl), out.data_ptr(), dst_off.data_ptr(),
                                             st.data_ptr(), scratch.data_ptr(), read_work.data_ptr(), work.data_ptr(), stream(torch))
        assert rc == 0, z.ST_NAMES.get(rc, rc)
        return [out, st, scratch]
    rb = (L.zmt_zstd_range_read_workspace_bytes if zstd else L.zmt_lz4_range_read_workspace_bytes)(ctypes.byref(pl))
    out, st, _ = twice(torch, [wb, rb], read, init=[state])
    assert not st.cpu().numpy().any()
    got, do = out.cpu().numpy(), dst_off.cpu().numpy()
    for r, (s, k) in enumerate(ranges):
        assert np.array_equal(got[do[r]: do[r] + k], src[s: s + k]), r
