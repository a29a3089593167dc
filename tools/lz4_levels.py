"""Speed and ratio of the LZ4 levels on one GPU, next to the reference at the same levels.

    python tools/lz4_levels.py [--gib 1] [--levels 1,10,11,12] [--chunk-mib 4] [--steps 3] [--ref-gib 0.25] [--out FILE]

Per level and input (GEN_TEXT, GEN_MIX), in chunks of `chunk-mib` (4 MiB: the reference's default for LZ4):
  - device-timed compress throughput of zmt_lz4_compress_level_device (CUDA events, one warm-up call, `steps` timed calls);
  - per-kernel times from zmt_prof_begin / zmt_prof_end over one further call;
  - ratio, and device-timed throughput of zmt_lz4_decompress_device on the frames just written;
  - the reference's LZ4MT_compressCCtx (oracle/_ref: the unmodified wrapper + liblz4, whose levels 3 and up run LZ4HC) on
    all host threads, on the first `ref-gib` of the same input, with its ratio.
The card's name and power limit are read in the same run.  One JSON line per run goes to stdout; --out also writes all of
them, with the card, to one JSON file."""
import argparse
import ctypes
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

KERNELS = {0: "lz4_blocks_pipe_kernel", 1: "xxh32_kernel", 2: "lz4_frame_sizes_kernel", 3: "scan_u64_kernel", 4: "lz4_frame_pack_kernel",
           11: "zstd_lazy_hash_kernel", 12: "radix sort + zstd_lazy_prev_kernel", 13: "zstd_lazy_search_kernel", 15: "lz4_hc_blocks_kernel"}


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


def profile(torch, fn):
    L = z.lib()
    L.zmt_prof_begin.restype = None
    L.zmt_prof_end.restype = ctypes.c_int
    ms, cnt = (ctypes.c_double * 16)(), (ctypes.c_int * 16)()
    L.zmt_prof_begin(); fn(); torch.cuda.synchronize(); L.zmt_prof_end(ms, cnt, 16)
    return {KERNELS[i]: round(ms[i], 3) for i in KERNELS if cnt[i]}


def reference(src, level, chunk):
    import _oracle as o
    if not o.have_ref():
        return None
    threads = os.cpu_count() or 1
    cap = src.size + src.size // 64 + (64 << 20)
    out = np.empty(cap, np.uint8); st = (ctypes.c_size_t * 5)()
    t = time.perf_counter()
    rc = o.ref().ref_lz4_compress_mem(threads, level, chunk, src.ctypes.data, src.size, out.ctypes.data, cap, st)
    dt = time.perf_counter() - t
    return None if rc else {"threads": threads, "gbps": round(src.size / dt / 1e9, 3), "ratio": round(src.size / st[0], 4), "bytes": int(src.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--levels", default="1,10,11,12")
    ap.add_argument("--chunk-mib", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--ref-gib", type=float, default=0.25)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.cuda.set_device(0)
    n, chunk = int(a.gib * (1 << 30)), a.chunk_mib << 20
    res = {"card": card(), "bytes": n, "chunk": chunk, "runs": []}
    print("card:", res["card"], flush=True)
    for kind, kname in ((z.GEN_TEXT, "text"), (z.GEN_MIX, "mix")):
        src = z.gen_stream(kind, n, chunk)
        d_in = torch.from_numpy(src).cuda()
        for level in [int(x) for x in a.levels.split(",")]:
            comp = z.Lz4DeviceCompressor(n, chunk, level=level)
            run = lambda: comp.run(d_in)
            ms = timed(torch, run, a.steps)
            kms = profile(torch, run)
            out, foff = comp.run(d_in); torch.cuda.synchronize()
            foff_h = foff.cpu().numpy()
            framed = out[: int(foff_h[-1])].cpu().numpy()
            offs, sizes = z.scan_frames(framed)
            dec = z.Lz4DeviceDecompressor(offs, sizes, [min(chunk, n - i) for i in range(0, n, chunk)])
            d_fr = torch.from_numpy(framed).cuda()
            dms = timed(torch, lambda: dec.run(d_fr), a.steps)
            dout, status = dec.run(d_fr); torch.cuda.synchronize()
            ok = not status.cpu().numpy().any() and torch.equal(dout[:n], d_in)
            r = {"input": kname, "level": level, "chunk": chunk, "ratio": round(n / framed.size, 4), "compress_gbps": round(n / ms / 1e6, 2),
                 "compress_ms": round(ms, 2), "kernel_ms": kms, "decompress_gbps": round(n / dms / 1e6, 2), "roundtrip_ok": bool(ok),
                 "reference": reference(src[: int(a.ref_gib * (1 << 30))], level, chunk)}
            print(json.dumps(r), flush=True)
            res["runs"].append(r)
            del comp, dec, d_fr, dout, out
            torch.cuda.empty_cache()
        del d_in
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
