import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import zstdmt_b200 as z, _oracle as o
import importlib.util
seed = int(sys.argv[1]); want_round = int(sys.argv[2])
# re-run the stress generator deterministically up to the failing round (same draws as tools/stress_gpu.py)
src_code = open(os.path.join(ROOT, "tools", "stress_gpu.py")).read()
pre = src_code[: src_code.index("t_end = time.time()")].replace("budget = float(sys.argv[1]) if len(sys.argv) > 1 else 60", "budget = 0").replace("seed = int(sys.argv[2]) if len(sys.argv) > 2 else 1", "seed = %d" % seed)
ns = {"__file__": os.path.join(ROOT, "tools", "stress_gpu.py"), "__name__": "stress_pre"}; exec(compile(pre, "stress_pre", "exec"), ns)
rng = ns["rng"]; recipe = ns["recipe"]
for r in range(want_round + 1):
    n = int(rng.choice([0, 1, 13, 5000, 65536, 65537, 1 << 20, (3 << 20) + 17, (9 << 20) + 1, 20 << 20]))
    n = max(0, n + int(rng.integers(-3, 4)) if n > 3 else n)
    chunk = int(rng.choice([65536, 100000, 1 << 20, 4 << 20, (1 << 20) + 4096]))
    src = recipe(n) if n else np.empty(0, np.uint8)
print("round", want_round, "n", n, "chunk", chunk)
torch.cuda.set_device(0)
bad = None
for ci in range(-(-n // chunk)):
    part = src[ci * chunk: (ci + 1) * chunk]
    zc = z.ZstdDeviceCompressor(part.size, chunk); zo, zf = zc.run(torch.from_numpy(part).cuda()); torch.cuda.synchronize()
    g = zo[: int(zf[-1])].cpu().numpy()
    rc, back = o.orc_decode(o.CODEC_ZSTD, g, part.size)
    ok = rc == 0 and np.array_equal(back, part)
    print("chunk", ci, "size", part.size, "->", g.size, "oracle rc", rc, "ok", ok)
    if not ok and bad is None:
        bad = ci
        os.makedirs(os.path.join(ROOT, "debug_out"), exist_ok=True)
        part.tofile(os.path.join(ROOT, "debug_out", "bad_src.bin")); g.tofile(os.path.join(ROOT, "debug_out", "bad_framed.bin"))
        if o.have_ref():
            rc2, b2, _ = o.ref_decompress(o.CODEC_ZSTD, g, part.size, threads=1); print("  libzstd rc", rc2, "ok", rc2 == 0 and np.array_equal(b2, part))
print("first bad chunk", bad)
