"""Cost of building the decoders' tables on the GPU (the device frame index) against the host path it replaces.

    python tools/frame_index_probe.py [--gib 1] [--steps 5] [--out FILE]

Streams, written on the GPU from GEN_MIX input: LZ4 level 1 and zstd level 3 in 1 MiB and 4 MiB chunks, zstd level 9 at
its default chunk (4 MiB); where oracle/_ref exists, also libzstd-written frames (the reference wrapper at level 3, 1 MiB
chunks, on the first quarter of the input).  Per stream:
  - index_ms: the device index (index call, and for zstd the block pass), CUDA events over `steps` calls;
  - kernels_ms: the same split by kernel (container walk, frame pass, scans, summary, block pass), from torch.profiler
    over one further call;
  - decode_ms: the decode call on the device-built tables, CUDA events;
  - host_ms: the host path the index replaces: D2H of the stream into pinned memory, the host header walk
    (scan_frames + the LZ4F content size, or zmt_zstd_scan_frame_host per frame) and the H2D of the tables;
  - identical: the decoded bytes from device-built and host-built tables are the same.
The card's name and power limit are read in the same run.  One JSON line per stream goes to stdout; --out writes all of
them, with the card, to one JSON file.

    python tools/frame_index_probe.py --plain [--gib 1] [--steps 5] [--out FILE]

Plain streams (.lz4 / .zst files: codec frames back to back, no container headers), each `gib` of GEN_MIX written by
liblz4 / libzstd on the host: one liblz4 streaming frame with 64 KiB linked blocks, one with 4 MiB independent blocks
and a content checksum, one libzstd streaming frame at level 3 with a checksum, and 1 MiB frames back to back for each
codec.  Per stream:
  - index_ms: the plain index call (zmt_{lz4,zstd}_index_plain_device), and for zstd the block pass, CUDA events;
  - kernels_ms: walk, tail, scans, summary and block pass, from torch.profiler over one further call;
  - decode_ms: the decode call on the device-built tables, CUDA events;
  - callback_ms: the host plain path on the same bytes: LZ4MT_ / ZSTDCB_decompressDCtx from memory to memory, wall clock;
  - identical: the device decode and the callback API both give the source bytes."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zstdmt_b200 as z  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().split("\n")[0] if r.returncode == 0 else "unknown"


def timed(torch, fn, steps):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def kernel_split(torch, fn, reps=1):
    """Device time per kernel group of one fn() call, the mean over `reps` profiled calls."""
    from torch.profiler import ProfilerActivity, profile
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    groups = {"walk": "zidx_walk_kernel", "frames": "_frames_kernel", "scan": "DeviceScan", "summary": "zidx_summary_kernel",
              "blocks": "zidx_zstd_blocks_kernel", "plain_walk": "zidx_plain_walk_kernel", "tail": "zidx_plain_tail_kernel"}
    out = {k: 0.0 for k in groups}
    for e in prof.events():
        for k, pat in groups.items():
            if pat in e.name and str(e.device_type).endswith("CUDA"):
                out[k] += (e.time_range.end - e.time_range.start) / 1000.0
    return {k: round(v / reps, 4) for k, v in out.items()}


class Tables:
    """Preallocated arguments of the index calls, so that the timed calls are only the enqueued work."""

    def __init__(self, torch, d, zstd, nframes, nblocks=0, plain=False):
        L = z.lib()
        e = lambda n, dt: torch.empty(max(n, 1), dtype=dt, device="cuda")
        self.d, self.zstd, self.n, self.nblocks = d, zstd, nframes, nblocks
        self.pad = z.PLAIN_PAD if plain else 0
        self.zidx = L.zmt_zstd_index_plain_device if plain else L.zmt_zstd_index_device
        self.lidx = L.zmt_lz4_index_plain_device if plain else L.zmt_lz4_index_device
        self.off, self.cs, self.oo = e(nframes, torch.int64), e(nframes, torch.int32), e(nframes + 1, torch.int64)
        self.first, self.scr, self.exp, self.seq = e(nframes + 1, torch.int32), e(nframes + 1, torch.int64), e(nframes, torch.int64), e(nframes, torch.int32)
        self.blocks = e(nblocks * L.zmt_zstd_blk_desc_bytes(), torch.uint8)
        self.work = e(L.zmt_index_workspace_bytes(nframes), torch.uint8)
        self.info = e(40, torch.uint8)

    def __call__(self):
        import torch
        L, s = z.lib(), torch.cuda.current_stream().cuda_stream
        if self.zstd:
            self.zidx(self.d.data_ptr(), self.d.numel(), self.n, self.off.data_ptr(), self.cs.data_ptr(), self.first.data_ptr(),
                      self.scr.data_ptr(), self.exp.data_ptr(), self.seq.data_ptr(), self.oo.data_ptr(), self.info.data_ptr(),
                      self.work.data_ptr(), s)
            L.zmt_zstd_blocks_device(self.d.data_ptr() - self.pad, self.n, self.off.data_ptr(), self.cs.data_ptr(), self.first.data_ptr(),
                                     self.scr.data_ptr(), self.blocks.data_ptr(), self.nblocks, s)
        else:
            self.lidx(self.d.data_ptr(), self.d.numel(), self.n, self.off.data_ptr(), self.cs.data_ptr(), self.oo.data_ptr(),
                      self.info.data_ptr(), self.work.data_ptr(), s)


def host_path(torch, d, zstd):
    """D2H of the stream, host walk, H2D of the tables; returns (ms, host-built decoder)."""
    h = torch.empty(d.numel(), dtype=torch.uint8, pin_memory=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    h.copy_(d); torch.cuda.synchronize()
    t1 = time.perf_counter()
    fb = h.numpy()
    if zstd:
        dec = z.ZstdDeviceDecompressor(fb)                                  # host scan + H2D of the tables, as the pipeline
        tab = [dec.d_blocks, dec.d_first, dec.d_expect, dec.d_fseq, dec.d_out_off]
    else:
        offs, sizes = z.scan_frames(fb)
        room = [int.from_bytes(fb[int(o) + 18: int(o) + 26].tobytes(), "little") if fb[int(o) + 16] & 8 else None for o in offs]
        if any(r is None for r in room):
            room = None
        dec = z.Lz4DeviceDecompressor(offs, sizes, room) if room is not None else None
        tab = [dec.d_off, dec.d_cs, dec.d_out_off] if dec is not None else []
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return {"d2h_ms": round((t1 - t0) * 1e3, 3), "scan_and_h2d_ms": round((t2 - t1) * 1e3, 3), "host_ms": round((t2 - t0) * 1e3, 3),
            "table_bytes": int(sum(t.numel() * t.element_size() for t in tab))}, dec


def probe(torch, name, d, zstd, steps):
    cls = z.ZstdDeviceDecompressor if zstd else z.Lz4DeviceDecompressor
    dev = cls.from_device(d)
    info = dev.index_info
    tabs = Tables(torch, d, zstd, info.nframes, info.nblocks if zstd else 0)
    rec = {"stream": name, "bytes": d.numel(), "frames": info.nframes, "blocks": info.nblocks, "out_bytes": info.out_bytes}
    rec["index_ms"] = round(timed(torch, tabs, steps), 4)
    rec["kernels_ms"] = kernel_split(torch, tabs)
    rec["decode_ms"] = round(timed(torch, lambda: dev.run(d), steps), 4)
    hp, hdec = host_path(torch, d, zstd)
    rec.update(hp)
    if hdec is not None:
        a, _ = dev.run(d); a = a.clone()
        b, _ = hdec.run(d)
        torch.cuda.synchronize()
        rec["identical"] = bool(dev.out_total == hdec.out_total and torch.equal(a[: dev.out_total], b[: hdec.out_total]) and
                                not dev.status[: info.nframes].any().item())
    return rec


def plain_streams(n, tmp):
    """(name, codec, stream bytes) of the plain streams, each of n bytes of GEN_MIX (gen_stream with 1 MiB chunks)."""
    from test_gpu_plain_segments import write_lz4_stream_prefs
    from test_gpu_plain_streams import lz4f, zstd1, zstd_adv
    mib = 1 << 20
    for name, kw in (("lz4-1frame-64KiB-linked", dict(blockSizeID=4, blockMode=0)),
                     ("lz4-1frame-4MiB-indep", dict(blockSizeID=7, blockMode=1, contentChecksumFlag=1))):
        path = os.path.join(tmp, "s.lz4")
        write_lz4_stream_prefs(path, n, kw)
        yield name, "lz4", np.fromfile(path, np.uint8)
        os.remove(path)
    src = z.gen_stream(z.GEN_MIX, n, mib)
    yield "zstd-1frame-l3-checksum", "zstd", zstd_adv(src, level=3, checksum=1, content_size=0, pieces=[8 * mib] * (n // (8 * mib)))
    yield "lz4-1MiB-frames", "lz4", np.concatenate([lz4f(src[i: i + mib], contentSize=min(mib, n - i)) for i in range(0, n, mib)])
    yield "zstd-1MiB-frames-l3", "zstd", np.concatenate([zstd1(src[i: i + mib], 3) for i in range(0, n, mib)])


def probe_plain(torch, name, codec, fb, src, steps):
    zstd = codec == "zstd"
    d = torch.from_numpy(fb).cuda()
    cls = z.ZstdDeviceDecompressor if zstd else z.Lz4DeviceDecompressor
    dev = cls.from_device(d, plain=True)
    info = dev.index_info
    tabs = Tables(torch, d, zstd, info.nframes, info.nblocks if zstd else 0, plain=True)
    rec = {"stream": name, "bytes": d.numel(), "frames": info.nframes, "blocks": info.nblocks, "out_bytes": info.out_bytes}
    rec["index_ms"] = round(timed(torch, tabs, steps), 4)
    rec["kernels_ms"] = kernel_split(torch, tabs, reps=steps)
    rec["decode_ms"] = round(timed(torch, lambda: dev.run(d), steps), 4)
    out, st = dev.run(d)
    torch.cuda.synchronize()
    oo, sz = dev.d_out_off[: info.nframes + 1].cpu().numpy(), dev.out_size[: info.nframes].cpu().numpy()
    got = torch.cat([out[int(oo[i]): int(oo[i]) + int(sz[i])] for i in range(info.nframes)]).cpu().numpy() if info.nframes else np.zeros(0, np.uint8)
    same = not st[: info.nframes].any().item() and np.array_equal(got, src)
    del out, got, d
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    rc, back, _ = z.decompress_mem(z.CODEC_ZSTD if zstd else z.CODEC_LZ4, fb, src.size + 16, threads=4)
    rec["callback_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    rec["identical"] = bool(same and rc == 0 and np.array_equal(back, src))
    return rec


def main_plain(a, torch, dev_card):
    import tempfile
    n = int(a.gib * (1 << 30)) // (8 << 20) * (8 << 20)
    src = z.gen_stream(z.GEN_MIX, n, 1 << 20)
    runs = []
    with tempfile.TemporaryDirectory() as tmp:
        for name, codec, fb in plain_streams(n, tmp):
            rec = probe_plain(torch, name, codec, fb, src, a.steps)
            rec["card"] = dev_card
            print(json.dumps(rec), flush=True)
            runs.append(rec)
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--plain", action="store_true", help="plain .lz4 / .zst streams through the plain index")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    dev_card = card()
    if a.plain:
        runs = main_plain(a, torch, dev_card)
        if a.out:
            with open(a.out, "w") as f:
                json.dump({"card": dev_card, "runs": runs}, f, indent=1)
        return
    n = int(a.gib * (1 << 30))
    src = torch.from_numpy(z.gen_stream(z.GEN_MIX, n, 1 << 20)).cuda()
    runs = []
    for codec, level, chunk in (("lz4", 1, 1 << 20), ("lz4", 1, 4 << 20), ("zstd", 3, 1 << 20), ("zstd", 3, 4 << 20), ("zstd", 9, 4 << 20)):
        comp = (z.Lz4DeviceCompressor if codec == "lz4" else z.ZstdDeviceCompressor)(n, chunk, level=level)
        out, foff = comp.run(src)
        total = int(foff[-1])
        d = out[:total].clone()
        del comp, out
        torch.cuda.empty_cache()
        rec = probe(torch, "%s-l%d-%dMiB" % (codec, level, chunk >> 20), d, codec == "zstd", a.steps)
        rec["card"] = dev_card
        print(json.dumps(rec), flush=True)
        runs.append(rec)
        del d
        torch.cuda.empty_cache()
    import _oracle as o
    if o.have_ref():
        m = n // 4
        rc, fb, _ = o.ref_compress(o.CODEC_ZSTD, src[:m].cpu().numpy(), threads=os.cpu_count() or 4, level=3, chunk=1 << 20)
        if rc == 0:
            rec = probe(torch, "libzstd-l3-1MiB", torch.from_numpy(fb).cuda(), True, a.steps)
            rec["card"] = dev_card
            print(json.dumps(rec), flush=True)
            runs.append(rec)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": dev_card, "runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
