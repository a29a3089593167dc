"""Many small zstd frames written against one dictionary: GPU decode (index + block table + decode, from a plain stream in
HBM) against libzstd's ZSTD_decompress_usingDDict on the host's threads.

python tools/zstd_dict_probe.py [MiB of records] [level]     (default 256 MiB, level 3; records of 1-4 KiB, 110 KiB dictionary)
Prints the card's name and power limit with one JSON line per measurement."""
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import ctypes.util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import zstdmt_b200 as z
import _zdict as zd

mib = int(sys.argv[1]) if len(sys.argv) > 1 else 256
level = int(sys.argv[2]) if len(sys.argv) > 2 else 3
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip() \
    if shutil.which("nvidia-smi") else "no nvidia-smi"
print("gpu:", q, flush=True)

d = zd.train(1, 110 << 10, nrec=2000)
base = zd.records(2, 4000, 1024, 4096)
rng = np.random.default_rng(3)
recs, total = [], 0
while total < (mib << 20):                              # records drawn from a pool, each with a few bytes changed
    r = base[int(rng.integers(0, len(base)))].copy()
    r[rng.integers(0, r.size, 4)] = rng.integers(48, 58, 4)
    recs.append(r); total += r.size
t0 = time.time()
L = zd.zstd()
frames = [zd.compress(r, d, level=level) for r in recs]
stream = np.concatenate(frames)
print("records %d, %.1f MiB -> %.1f MiB compressed (ratio %.2f), libzstd level %d compress %.1f s"
      % (len(recs), total / 2**20, stream.size / 2**20, total / stream.size, level, time.time() - t0), flush=True)

dct = z.ZstdDictionary(d)
d_in = torch.from_numpy(stream).cuda()
ev = lambda: torch.cuda.Event(enable_timing=True)
# whole route: device index, block table, decode
for it in range(4):
    a, b = ev(), ev()
    a.record()
    dec = z.ZstdDeviceDecompressor.from_device(d_in, plain=True, dictionary=dct, max_frames=len(frames))
    out, st = dec.run(d_in)
    b.record(); torch.cuda.synchronize()
    route_ms = a.elapsed_time(b)
assert int(st.abs().sum()) == 0
oo = dec.d_out_off.cpu().numpy()
assert all(np.array_equal(out[int(oo[i]): int(oo[i]) + recs[i].size].cpu().numpy(), recs[i]) for i in range(0, len(recs), max(1, len(recs) // 500)))
assert int(oo[-1]) + 0 <= dec.out.numel() and dec.out_total == total
# decode alone, tables built once
times = []
for it in range(10):
    a, b = ev(), ev()
    a.record(); dec.run(d_in); b.record(); torch.cuda.synchronize()
    times.append(a.elapsed_time(b))
dec_ms = sorted(times)[len(times) // 2]
print(json.dumps({"what": "gpu decode", "frames": len(recs), "content_mib": round(total / 2**20, 1), "decode_ms": round(dec_ms, 3),
                  "decode_GBps": round(total / dec_ms / 1e6, 2), "index_and_decode_ms": round(route_ms, 3)}), flush=True)

# libzstd on the host's threads, one ZSTD_DDict shared by all: a small C loop (built into a temporary directory), so the
# figure is libzstd's and not the cost of one Python call per frame
C_SRC = r"""
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
void* ZSTD_createDCtx(void); size_t ZSTD_freeDCtx(void*); unsigned ZSTD_isError(size_t);
size_t ZSTD_decompress_usingDDict(void*, void*, size_t, const void*, size_t, const void*);
typedef struct { const uint8_t* src; const int64_t* soff; uint8_t* dst; const int64_t* doff; const void* ddict; long n, k, nth, bad; } job;
static void* run(void* a) {
    job* j = (job*)a; void* dctx = ZSTD_createDCtx();
    for (long i = j->k; i < j->n; i += j->nth) {
        size_t r = ZSTD_decompress_usingDDict(dctx, j->dst + j->doff[i], j->doff[i + 1] - j->doff[i], j->src + j->soff[i], j->soff[i + 1] - j->soff[i], j->ddict);
        if (ZSTD_isError(r) || (int64_t)r != j->doff[i + 1] - j->doff[i]) j->bad++;
    }
    ZSTD_freeDCtx(dctx); return 0;
}
long decode_all(const uint8_t* src, const int64_t* soff, uint8_t* dst, const int64_t* doff, const void* ddict, long n, long nth) {
    pthread_t t[256]; job j[256]; long bad = 0;
    for (long k = 0; k < nth; k++) { job x = { src, soff, dst, doff, ddict, n, k, nth, 0 }; j[k] = x; pthread_create(&t[k], 0, run, &j[k]); }
    for (long k = 0; k < nth; k++) { pthread_join(t[k], 0); bad += j[k].bad; }
    return bad;
}
"""
tmp = tempfile.mkdtemp(prefix="zdict_probe_")
with open(os.path.join(tmp, "h.c"), "w") as f:
    f.write(C_SRC)
libz = ctypes.util.find_library("zstd") or "libzstd.so.1"
libz = next((os.path.join(d_, "libzstd.so.1") for d_ in ("/usr/lib/x86_64-linux-gnu", "/usr/lib64", "/usr/lib")
             if os.path.exists(os.path.join(d_, "libzstd.so.1"))), libz)
subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-pthread", "-o", os.path.join(tmp, "h.so"), os.path.join(tmp, "h.c"), libz], check=True)
H = ctypes.CDLL(os.path.join(tmp, "h.so"))
H.decode_all.restype = ctypes.c_long
H.decode_all.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_long, ctypes.c_long]
L.ZSTD_createDDict.restype = ctypes.c_void_p; L.ZSTD_createDDict.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
dd = np.ascontiguousarray(d)
ddict = L.ZSTD_createDDict(dd.ctypes.data, dd.size)
offs = np.zeros(len(frames) + 1, np.int64); offs[1:] = np.cumsum([f.size for f in frames])
ooff = np.zeros(len(recs) + 1, np.int64); ooff[1:] = np.cumsum([r.size for r in recs])
dst = np.empty(total, np.uint8)
nth = min(os.cpu_count() or 1, 256)
best = None
for it in range(3):
    t0 = time.time()
    bad = H.decode_all(stream.ctypes.data, offs.ctypes.data, dst.ctypes.data, ooff.ctypes.data, ddict, len(frames), nth)
    el = time.time() - t0
    assert bad == 0
    best = el if best is None or el < best else best
assert np.array_equal(dst[: recs[0].size], recs[0]) and np.array_equal(dst[-recs[-1].size:], recs[-1])
shutil.rmtree(tmp)
print(json.dumps({"what": "libzstd ZSTD_decompress_usingDDict", "threads": nth, "ms": round(best * 1e3, 1),
                  "GBps": round(total / best / 1e9, 2)}), flush=True)
