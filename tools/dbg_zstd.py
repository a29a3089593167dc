import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import zstdmt_b200 as z, _oracle as o
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 20
kind = int(sys.argv[2]) if len(sys.argv) > 2 else z.GEN_MIX
first = int(sys.argv[3]) if len(sys.argv) > 3 else 0
chunk = 1 << 20
src = z.gen_stream(kind, n, chunk, first=first)
d_in = torch.from_numpy(src).cuda() if n else torch.empty(1, dtype=torch.uint8, device="cuda")
comp = z.ZstdDeviceCompressor(n, chunk)
out, foff = comp.run(d_in)
torch.cuda.synchronize()
f = out[: int(foff[-1])].cpu().numpy()
print("n", n, "->", f.size, "ratio %.3f" % (n / max(1, f.size)), "head", f[:24].tobytes().hex())
rc, back = o.orc_decode(o.CODEC_ZSTD, f, n)
print("oracle decode rc", rc, "ok", back.size == n and np.array_equal(back, src))
if rc != 0 or not np.array_equal(back, src):
    os.makedirs(os.path.join(ROOT, "debug_out"), exist_ok=True)
    f.tofile(os.path.join(ROOT, "debug_out", "bad_framed.bin")); src.tofile(os.path.join(ROOT, "debug_out", "bad_src.bin"))
if o.have_ref():
    for T in (1, 3):
        rc, b2, st = o.ref_decompress(o.CODEC_ZSTD, f, n, threads=T)
        print("libzstd (reference T=%d) rc %d ok %s" % (T, rc, b2.size == n and np.array_equal(b2, src)))
dec = z.ZstdDeviceDecompressor(f)
print("scan", set(dec.scan_status), "frames", dec.n, "blocks", dec.nblk)
d_f = torch.from_numpy(f).cuda()
dout, st = dec.run(d_f); torch.cuda.synchronize()
print("GPU decode status", st.cpu().unique().tolist(), "ok", dec.out_total == n and np.array_equal(dout[:n].cpu().numpy(), src))
# callback API both ways
rc, fr2, stt = z.compress_mem(z.CODEC_ZSTD, src, threads=4, level=3, chunk=chunk)
print("ZSTDCB_compressCCtx rc", rc, "same bytes as device path", fr2.size == f.size and np.array_equal(fr2, f), stt)
rc, bk, stt = z.decompress_mem(z.CODEC_ZSTD, fr2, n + 16, threads=4)
print("ZSTDCB_decompressDCtx rc", rc, "ok", bk.size == n and np.array_equal(bk, src), stt)
if os.environ.get("TIME"):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2): comp.run(d_in)
    e0.record()
    for _ in range(5): comp.run(d_in)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    print("compress ms/step %.3f  in GB/s %.1f" % (ms, n / ms / 1e6))
    for _ in range(2): dec.run(d_f)
    e0.record()
    for _ in range(5): dec.run(d_f)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    print("decompress ms/step %.3f  out GB/s %.1f" % (ms, n / ms / 1e6))
