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
them, with the card, to one JSON file."""
import argparse
import json
import os
import subprocess
import sys
import time


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


def kernel_split(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    groups = {"walk": "zidx_walk_kernel", "frames": "_frames_kernel", "scan": "DeviceScan", "summary": "zidx_summary_kernel",
              "blocks": "zidx_zstd_blocks_kernel"}
    out = {k: 0.0 for k in groups}
    for e in prof.events():
        for k, pat in groups.items():
            if pat in e.name and str(e.device_type).endswith("CUDA"):
                out[k] += (e.time_range.end - e.time_range.start) / 1000.0
    return {k: round(v, 4) for k, v in out.items()}


class Tables:
    """Preallocated arguments of the index calls, so that the timed calls are only the enqueued work."""

    def __init__(self, torch, d, zstd, nframes, nblocks=0):
        L = z.lib()
        e = lambda n, dt: torch.empty(max(n, 1), dtype=dt, device="cuda")
        self.d, self.zstd, self.n, self.nblocks = d, zstd, nframes, nblocks
        self.off, self.cs, self.oo = e(nframes, torch.int64), e(nframes, torch.int32), e(nframes + 1, torch.int64)
        self.first, self.scr, self.exp, self.seq = e(nframes + 1, torch.int32), e(nframes + 1, torch.int64), e(nframes, torch.int64), e(nframes, torch.int32)
        self.blocks = e(nblocks * L.zmt_zstd_blk_desc_bytes(), torch.uint8)
        self.work = e(L.zmt_index_workspace_bytes(nframes), torch.uint8)
        self.info = e(40, torch.uint8)

    def __call__(self):
        import torch
        L, s = z.lib(), torch.cuda.current_stream().cuda_stream
        if self.zstd:
            L.zmt_zstd_index_device(self.d.data_ptr(), self.d.numel(), self.n, self.off.data_ptr(), self.cs.data_ptr(), self.first.data_ptr(),
                                    self.scr.data_ptr(), self.exp.data_ptr(), self.seq.data_ptr(), self.oo.data_ptr(), self.info.data_ptr(),
                                    self.work.data_ptr(), s)
            L.zmt_zstd_blocks_device(self.d.data_ptr(), self.n, self.off.data_ptr(), self.cs.data_ptr(), self.first.data_ptr(), self.scr.data_ptr(),
                                     self.blocks.data_ptr(), self.nblocks, s)
        else:
            L.zmt_lz4_index_device(self.d.data_ptr(), self.d.numel(), self.n, self.off.data_ptr(), self.cs.data_ptr(), self.oo.data_ptr(),
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    dev_card = card()
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
