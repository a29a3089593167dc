"""Small decode workloads for compute-sanitizer (memcheck / racecheck): LZ4 own + reference-framed (linked) streams, zstd own +
libzstd-framed streams, through the device API and the callback API; a libzstd frame decoded as segments through the device
API and through the callback API in 1 MiB batches; zstd frames written against a dictionary through the host scan and the
device index.  python tools/sanitize_decode.py [MiB]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import zstdmt_b200 as z, _oracle as o
mib = int(sys.argv[1]) if len(sys.argv) > 1 else 6
chunk, n = 1 << 20, (mib << 20) + 12345
src = z.gen_stream(z.GEN_MIX, n, chunk)
d_src = torch.from_numpy(src).cuda()
outs = [min(chunk, n - i * chunk) for i in range(-(-n // chunk))]
def lz4_dec(framed, label):
    offs, sizes = z.scan_frames(framed)
    dec = z.Lz4DeviceDecompressor(offs, sizes, outs)
    out, st = dec.run(torch.from_numpy(framed).cuda()); torch.cuda.synchronize()
    assert int(st.abs().sum()) == 0 and torch.equal(out[:n], d_src), label
    print(label, "ok", flush=True)
def zstd_dec(framed, label):
    dec = z.ZstdDeviceDecompressor(framed)
    out, st = dec.run(torch.from_numpy(framed).cuda()); torch.cuda.synchronize()
    assert int(st.abs().sum()) == 0 and torch.equal(out[:n], d_src), label
    print(label, "ok", flush=True)
c = z.Lz4DeviceCompressor(n, chunk); out, foff = c.run(d_src); torch.cuda.synchronize()
lz4_dec(out[: int(foff[-1])].cpu().numpy(), "lz4 own stream")
rc, rf, _ = o.ref_compress(o.CODEC_LZ4, src, threads=4, level=1, chunk=chunk); assert rc == 0
lz4_dec(rf, "lz4 reference-framed (linked blocks)")
zc = z.ZstdDeviceCompressor(n, chunk); zout, zf = zc.run(d_src); torch.cuda.synchronize()
zstd_dec(zout[: int(zf[-1])].cpu().numpy(), "zstd own stream")
rc, zrf, _ = o.ref_compress(o.CODEC_ZSTD, src, threads=4, level=3, chunk=chunk); assert rc == 0
zstd_dec(zrf, "zstd reference-framed (libzstd level 3)")
for codec, fr in ((z.CODEC_LZ4, rf), (z.CODEC_ZSTD, zrf)):
    rc, back, st = z.decompress_mem(codec, fr, n + 16, threads=4)
    assert rc == 0 and np.array_equal(back, src)
print("callback API ok")
# zstd segments: a libzstd frame (level 3, content checksum, no content size) cut at block boundaries, then as a plain
# stream in 1 MiB batches
from test_gpu_plain_streams import zstd_adv
from test_zstd_frame_segments import header_walk
zf1 = zstd_adv(src, 3, checksum=1, pieces=[n // 2, n - n // 2])
cuts = [a + k for a, k, _ in header_walk(zf1)["blocks"]][:-1]
back, st = z.zstd_decode_segments(zf1, cuts[:: max(1, len(cuts) // 6)])
assert st == 0 and np.array_equal(back, src)
os.environ["ZSTDMT_B200_PLAIN_MB"] = "1"
rc, back, st = z.decompress_mem(z.CODEC_ZSTD, zf1, n + 16, threads=4, inputsize=1 << 20)
assert rc == 0 and np.array_equal(back, src)
print("zstd segments ok")
# zstd frames written against a dictionary (formatted and raw content): host scan, device index of a container and of a
# plain stream
import _zdict as zd
recs = zd.records(5, 400)
for d, kind in ((zd.train(6, 64 << 10), zd.DCT_AUTO), (np.concatenate(zd.records(7, 20))[: 16 << 10], zd.DCT_RAW)):
    dct = z.ZstdDictionary(d)
    frames = [zd.compress(r, d, level=(1, 3, 19)[i % 3], checksum=i & 1, kind=kind) for i, r in enumerate(recs)]
    for fr, plain in ((zd.container(frames), False), (zd.plain(frames), True)):
        d_fr = torch.from_numpy(fr).cuda()
        decs = [z.ZstdDeviceDecompressor.from_device(d_fr, plain=plain, dictionary=dct)]
        if not plain:
            decs.append(z.ZstdDeviceDecompressor(fr, dictionary=dct))
        for dec in decs:
            out, st = dec.run(d_fr); torch.cuda.synchronize()
            oo = dec.d_out_off.cpu().numpy()
            assert int(st.abs().sum()) == 0 and all(np.array_equal(out[int(oo[i]): int(oo[i]) + r.size].cpu().numpy(), r) for i, r in enumerate(recs))
print("zstd dictionary ok")
