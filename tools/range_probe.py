"""Cost of range reads (RangeReader) against a whole-stream decode of the same stream.

    python tools/range_probe.py [--gib 1] [--steps 3] [--out FILE]

Streams, written on the GPU from `gib` GiB of GEN_MIX input: LZ4 level 1 and zstd level 3, each in 1 MiB and 4 MiB
chunks.  Each stream is indexed once (the RangeReader constructor: device index and content table).  Then per batch of
seeded random ranges, M = 1, 16, 256 and 4096 ranges of 4 KiB and one batch of 64 ranges of 1 MiB:
  - device_ms: CUDA events around one read() (plan, summary read-back, pack, decode, gather), the mean over `steps`;
  - wall_ms: host wall time of the same call, synchronised, summary read-back included;
  - decoded_mib: the content of the frames the batch decodes (the plan's scratch_bytes), and their count;
and, once per stream, the whole-stream decode (from_device tables, run()) for comparison.  The card's name and power
limit are read in the same run.  One JSON line per stream goes to stdout; --out writes them, with the card, to a file."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import zstdmt_b200 as z  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().split("\n")[0] if r.returncode == 0 else "unknown"


def timed(torch, fn, steps):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    n = int(a.gib * (1 << 30))
    src = torch.from_numpy(z.gen_stream(z.GEN_MIX, n, 1 << 20)).cuda()
    rows = []
    for codec, level in (("lz4", 1), ("zstd", 3)):
        for chunk in (1 << 20, 4 << 20):
            cls = z.Lz4DeviceCompressor if codec == "lz4" else z.ZstdDeviceCompressor
            c = cls(n, chunk, level=level)
            out, off = c.run(src)
            torch.cuda.synchronize()
            d = out[: int(off[c.nchunks].item())].clone()
            del c, out
            t0 = time.perf_counter()
            R = z.RangeReader(d, codec)
            torch.cuda.synchronize()
            index_ms = (time.perf_counter() - t0) * 1e3
            dec = (z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor).from_device(d)
            whole_ms = timed(torch, lambda: dec.run(d), a.steps)
            del dec
            rng = np.random.default_rng(7)
            batches = []
            for m, ln in ((1, 4096), (16, 4096), (256, 4096), (4096, 4096), (64, 1 << 20)):
                st = rng.integers(0, n - ln, size=m)
                ranges = torch.from_numpy(np.stack([st, np.full(m, ln)], 1).astype(np.int64)).cuda()
                got, _, status = R.read(ranges)
                torch.cuda.synchronize()
                ok = not status.any().item() and all(torch.equal(got[i * ln:(i + 1) * ln], src[int(s): int(s) + ln]) for i, s in enumerate(st[:8]))
                dev_ms = timed(torch, lambda: R.read(ranges), a.steps)
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    R.read(ranges)
                    torch.cuda.synchronize()
                wall_ms = (time.perf_counter() - t0) * 1e3 / a.steps
                batches.append(dict(ranges=m, range_bytes=ln, frames=R.plan.nsel, decoded_mib=round(R.plan.scratch_bytes / 2**20, 1),
                                    device_ms=round(dev_ms, 3), wall_ms=round(wall_ms, 3), correct=bool(ok)))
            row = dict(codec=codec, level=level, chunk=chunk, frames=R.n, stream_mib=round(d.numel() / 2**20, 1), index_ms=round(index_ms, 2),
                       whole_decode_ms=round(whole_ms, 3), batches=batches)
            print(json.dumps(row), flush=True)
            rows.append(row)
            del R, d
            torch.cuda.empty_cache()
    res = dict(card=card(), gib=a.gib, rows=rows)
    print(json.dumps(dict(card=res["card"])))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
