"""Many small records compressed against one dictionary: the GPU (zmt_zstd_compress_dict_device, records of 1-4 KiB in
4 KiB slots) with and without the dictionary, the index build, and libzstd's ZSTD_compress_usingCDict on 8 host threads.

python tools/zstd_dict_compress_probe.py [MiB of records]     (default 256; levels 6, 9 and 12; 110 KiB trained dictionary)
Prints the card's name and power limit with one JSON line per measurement.  Ratios are record bytes over zstd frame bytes
(the 12-byte container headers of the GPU's frames excluded); GPU times are CUDA events, warmed up, median of 7."""
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import zstdmt_b200 as z
import _zdict as zd

mib = int(sys.argv[1]) if len(sys.argv) > 1 else 256
LEVELS, SLOT, NTH = (6, 9, 12), 4096, 8
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip() \
    if shutil.which("nvidia-smi") else "no nvidia-smi"
print("gpu:", q, flush=True)

d = zd.train(1, 110 << 10, nrec=2000)
base = zd.records(2, 4000, 1024, 4096)
rng = np.random.default_rng(3)
sizes, picks, total = [], [], 0
while total < (mib << 20):                              # records drawn from a pool, each with a few bytes changed
    k = int(rng.integers(0, len(base)))
    picks.append(k); sizes.append(base[k].size); total += base[k].size
n = len(sizes)
src = np.zeros(n * SLOT, np.uint8)
for i, k in enumerate(picks):
    r = src[i * SLOT: i * SLOT + sizes[i]]
    r[:] = base[k]
    r[rng.integers(0, r.size, 4)] = rng.integers(48, 58, 4)
cb = np.array(sizes, np.uint32)
print("records %d, %.1f MiB in %d-byte slots" % (n, total / 2**20, SLOT), flush=True)

d_in = torch.from_numpy(src).cuda()
d_cb = torch.from_numpy(cb.astype(np.int32)).cuda()
ev = lambda: torch.cuda.Event(enable_timing=True)


def timed(fn, reps=7, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = ev(), ev()
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


dct = z.ZstdDictionary(d)
L = z.lib()
cd = torch.empty(L.zmt_zstd_cdict_bytes(d.size), dtype=torch.uint8, device="cuda")
st = torch.cuda.current_stream().cuda_stream
build_ms = timed(lambda: L.zmt_zstd_cdict_build_device(dct.d_ddict.data_ptr(), d.size, cd.data_ptr(), st))
print(json.dumps({"what": "gpu index build", "dict_bytes": int(d.size), "ms": round(build_ms, 3)}), flush=True)

for level in LEVELS:
    for name, dic in (("gpu with dictionary", dct), ("gpu without dictionary", None)):
        comp = z.ZstdDeviceCompressor(src.size, SLOT, level=level, dictionary=dic)
        ms = timed(lambda: comp.run(d_in, chunk_bytes=d_cb))
        out, foff = comp.run(d_in, chunk_bytes=d_cb)
        torch.cuda.synchronize()
        fbytes = int(foff[-1].item()) - 12 * n
        if dic is not None:                              # spot-check frames against libzstd with the dictionary
            fo = foff.cpu().numpy()
            for i in range(0, n, max(1, n // 200)):
                fr = out[int(fo[i]) + 12: int(fo[i + 1])].cpu().numpy()
                bad, back = zd.decompress(fr, d, sizes[i])
                assert not bad and np.array_equal(back, src[i * SLOT: i * SLOT + sizes[i]])
        print(json.dumps({"what": name, "level": level, "ratio": round(total / fbytes, 3), "ms": round(ms, 2),
                          "GBps": round(total / ms / 1e6, 2)}), flush=True)
        del comp
        torch.cuda.empty_cache()

# libzstd on NTH host threads, one ZSTD_CDict per level shared by all: a small C loop (built into a temporary directory)
C_SRC = r"""
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
void* ZSTD_createCCtx(void); size_t ZSTD_freeCCtx(void*); unsigned ZSTD_isError(size_t);
size_t ZSTD_compress_usingCDict(void*, void*, size_t, const void*, size_t, const void*);
typedef struct { const uint8_t* src; const uint32_t* sz; long slot; uint8_t* dst; long cap; const void* cdict; long n, k, nth; long long bytes; long bad; } job;
static void* run(void* a) {
    job* j = (job*)a; void* cctx = ZSTD_createCCtx();
    for (long i = j->k; i < j->n; i += j->nth) {
        size_t r = ZSTD_compress_usingCDict(cctx, j->dst + i * j->cap, j->cap, j->src + i * j->slot, j->sz[i], j->cdict);
        if (ZSTD_isError(r)) j->bad++; else j->bytes += r;
    }
    ZSTD_freeCCtx(cctx); return 0;
}
long long compress_all(const uint8_t* src, const uint32_t* sz, long slot, uint8_t* dst, long cap, const void* cdict, long n, long nth) {
    pthread_t t[256]; job j[256]; long long bytes = 0; long bad = 0;
    for (long k = 0; k < nth; k++) { job x = { src, sz, slot, dst, cap, cdict, n, k, nth, 0, 0 }; j[k] = x; pthread_create(&t[k], 0, run, &j[k]); }
    for (long k = 0; k < nth; k++) { pthread_join(t[k], 0); bytes += j[k].bytes; bad += j[k].bad; }
    return bad ? -1 : bytes;
}
"""
tmp = tempfile.mkdtemp(prefix="zdict_cprobe_")
try:
    with open(os.path.join(tmp, "h.c"), "w") as f:
        f.write(C_SRC)
    libz = next((os.path.join(d_, "libzstd.so.1") for d_ in ("/usr/lib/x86_64-linux-gnu", "/usr/lib64", "/usr/lib")
                 if os.path.exists(os.path.join(d_, "libzstd.so.1"))), "libzstd.so.1")
    subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-pthread", "-o", os.path.join(tmp, "h.so"), os.path.join(tmp, "h.c"), libz], check=True)
    H = ctypes.CDLL(os.path.join(tmp, "h.so"))
    H.compress_all.restype = ctypes.c_longlong
    H.compress_all.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long, ctypes.c_void_p, ctypes.c_long, ctypes.c_void_p, ctypes.c_long, ctypes.c_long]
    Z = zd.zstd()
    Z.ZSTD_createCDict.restype = ctypes.c_void_p; Z.ZSTD_createCDict.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    Z.ZSTD_freeCDict.argtypes = [ctypes.c_void_p]
    cap = SLOT + 512
    dst = np.empty(n * cap, np.uint8)
    dd = np.ascontiguousarray(d)
    for level in LEVELS:
        cdict = Z.ZSTD_createCDict(dd.ctypes.data, dd.size, level)
        best = None
        for _ in range(3):
            t0 = time.time()
            fb = H.compress_all(src.ctypes.data, cb.ctypes.data, SLOT, dst.ctypes.data, cap, cdict, n, NTH)
            el = time.time() - t0
            assert fb > 0
            best = el if best is None or el < best else best
        Z.ZSTD_freeCDict(cdict)
        print(json.dumps({"what": "libzstd ZSTD_compress_usingCDict", "level": level, "threads": NTH, "ratio": round(total / fb, 3),
                          "ms": round(best * 1e3, 1), "GBps": round(total / best / 1e9, 2)}), flush=True)
finally:
    shutil.rmtree(tmp)
