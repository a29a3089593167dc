"""Plain .lz4 and .zst streams of one large frame through LZ4MT_decompressDCtx / ZSTDCB_decompressDCtx: the whole-frame
path against segments.

For each stream, decodes it twice, alternating, in a fresh subprocess each time:
  whole     ZSTDMT_B200_PLAIN_MB large enough to hold the frame: the frame is decoded in one batch
  segments  the default 64 MiB batches: the frame is decoded as a chain of segments
The streams, each one frame written by the codec library's streaming API:
  lz4_linked_64k         linked 64 KiB blocks (the lz4 CLI's default)
  lz4_indep_4m_cchk      independent 4 MiB blocks, content checksum
  zstd_l3_cchk           level 3, content checksum and content size (what the zstd CLI writes for a file)
  zstd_l3_w23            level 3 with an 8 MiB window (windowLog 23, level 19's; level 19 itself writes 4 GiB too slowly)
  zstd_l3_stream         level 3, content checksum, no content size (what `zstd < pipe` writes)
and prints one JSON line per run: GB/s of content from a host clock around the call (which returns synchronised),
the subprocess's peak RSS, and the device's used-memory high-water mark during the call (NVML, sampled every 5 ms by a
thread of the child; device_used_before_mib is the reading before the call).  Input is read from a file in a temporary directory,
output is discarded.  The card name and power limit are printed first.

    python tools/plain_stream_probe.py [--gib 4] [--runs 2] [--codec lz4|zstd|all]   (--runs: whole/segments pairs per stream)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

CHILD = r"""
import ctypes, json, resource, sys, threading, time
sys.path.insert(0, sys.argv[1])
import zstdmt_b200 as z
L = z.lib()
peak = [0]; stop = [False]
def sampler():
    try:
        nv = ctypes.CDLL("libnvidia-ml.so.1"); nv.nvmlInit_v2()
        h = ctypes.c_void_p(); nv.nvmlDeviceGetHandleByIndex_v2(0, ctypes.byref(h))
        class M(ctypes.Structure): _fields_ = [("total", ctypes.c_ulonglong), ("free", ctypes.c_ulonglong), ("used", ctypes.c_ulonglong)]
        m = M()
        while not stop[0]:
            if nv.nvmlDeviceGetMemoryInfo(h, ctypes.byref(m)) == 0: peak[0] = max(peak[0], m.used)
            time.sleep(0.005)
    except OSError:
        pass
f = open(sys.argv[2], "rb")
def rd(_, b):
    buf = (ctypes.c_char * b.contents.size).from_address(b.contents.buf)
    b.contents.size = f.readinto(buf); return 0
def wr(_, b): return 0
rdf, wrf = z.RW_FN(rd), z.RW_FN(wr)
rw = z.RdWr(rdf, None, wrf, None)
api = sys.argv[3]                                   # LZ4MT or ZSTDCB
ctx = getattr(L, api + "_createDCtx")(4, 1 << 20)
t = threading.Thread(target=sampler); t.start(); time.sleep(0.05); base = peak[0]
t0 = time.perf_counter()
rc = getattr(L, api + "_decompressDCtx")(ctx, ctypes.byref(rw))
dt = time.perf_counter() - t0
stop[0] = True; t.join()
out = getattr(L, api + "_GetOutsizeDCtx")(ctx)
getattr(L, api + "_freeDCtx")(ctx)
print(json.dumps(dict(rc=int(rc), out=int(out), seconds=dt, gbps=out / dt / 1e9, peak_rss_mib=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024,
                      device_used_peak_mib=peak[0] / 2**20, device_used_before_mib=base / 2**20)))
"""


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--codec", choices=["lz4", "zstd", "all"], default="all")
    a = ap.parse_args()
    from test_gpu_plain_segments import write_lz4_stream_prefs
    from test_gpu_zstd_segments import write_zstd_stream
    print(json.dumps({"card": card()}), flush=True)
    total = int(a.gib * (1 << 30))
    streams = []
    if a.codec in ("lz4", "all"):
        streams += [("lz4_linked_64k", "LZ4MT", lambda p: write_lz4_stream_prefs(p, total, dict(blockSizeID=4, blockMode=0))),
                    ("lz4_indep_4m_cchk", "LZ4MT", lambda p: write_lz4_stream_prefs(p, total, dict(blockSizeID=7, blockMode=1, contentChecksumFlag=1)))]
    if a.codec in ("zstd", "all"):
        streams += [("zstd_l3_cchk", "ZSTDCB", lambda p: write_zstd_stream(p, total, level=3, pledged=True)),
                    ("zstd_l3_w23", "ZSTDCB", lambda p: write_zstd_stream(p, total, level=3, pledged=True, window_log=23)),
                    ("zstd_l3_stream", "ZSTDCB", lambda p: write_zstd_stream(p, total, level=3))]
    with tempfile.TemporaryDirectory() as td:
        for name, api, write in streams:
            path = os.path.join(td, name)
            write(path)
            size = os.path.getsize(path)
            for r in range(a.runs):
                for mode, mb in (("whole", (size >> 20) + 64), ("segments", 64)):
                    env = dict(os.environ, ZSTDMT_B200_PLAIN_MB=str(mb))
                    p = subprocess.run([sys.executable, "-c", CHILD, ROOT, path, api], capture_output=True, text=True, env=env)
                    res = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else {"error": p.stderr[-500:]}
                    res.update(stream=name, mode=mode, plain_mb=mb, frame_bytes=size, run=r)
                    print(json.dumps(res), flush=True)
            os.remove(path)


if __name__ == "__main__":
    main()
