"""Where the LZ4 block compressor's cycles go, per team and phase (the table of DESIGN.md §3.4).  Needs a GPU.

    python tools/lz4_phase_probe.py [--gib 8] [--kind mix] [--lib PATH]

Builds the product library with -DZMT_PHASE_PROBE into build/phase_probe/ (or loads --lib), compresses the bench's
lz4-compress workload once to warm up and once measured (LZ4 level 1, synthetic Silesia-mix, 1 MiB chunks), and prints
each team's share of its own cycles per phase of lz4_blocks_pipe_kernel: clock64() deltas taken by thread 0 of each team,
summed over all CTAs.  The instrumented kernel is slower than the product; only the shares are meant to be compared.
"""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NPHASE = 8
ROWS = [("staging", "staging"), ("EMPTY wait", "FULL wait"), ("candidate rounds", "marking walk"), ("walk 0", "piece list"),
        ("walk 1", "head detection"), ("path resolution", "emission + long jobs"), ("FULL arrive", "EMPTY arrive"),
        ("final sync + last literals", "flush + final sync + last literals")]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gib", type=float, default=8.0)
    ap.add_argument("--kind", default="mix", choices=["mix", "text", "zeros", "random"])
    ap.add_argument("--lib", default=None, help="an already built probe library (default: build one into build/phase_probe/)")
    args = ap.parse_args()

    from zstdmt_b200 import build
    lib = args.lib or build.build_product(defines=["ZMT_PHASE_PROBE"], out_dir=os.path.join(ROOT, "build", "phase_probe"))
    import torch
    import zstdmt_b200 as z
    z.LIB_PATH = os.path.abspath(lib)                       # before the first z.lib(): load the probe library, not the product
    L = z.lib()
    take = L.zmt_phase_probe_take
    take.restype = ctypes.c_int
    take.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]

    chunk = 1 << 20
    n = int(args.gib * (1 << 30)) // chunk * chunk
    kind = {"mix": z.GEN_MIX, "text": z.GEN_TEXT, "zeros": z.GEN_ZEROS, "random": z.GEN_RANDOM}[args.kind]
    d_in = torch.from_numpy(z.gen_stream(kind, n, chunk)).cuda()
    comp = z.Lz4DeviceCompressor(n, chunk)
    cyc = (ctypes.c_ulonglong * (2 * NPHASE))()
    comp.run(d_in); torch.cuda.synchronize()
    assert take(cyc) == 0
    comp.run(d_in); torch.cuda.synchronize()
    assert take(cyc) == 0

    a, b = list(cyc[:NPHASE]), list(cyc[NPHASE:])
    ta, tb = sum(a), sum(b)
    print("%s: %s, %.2f GiB of %s, LZ4 level 1, 1 MiB chunks; share of each team's cycles"
          % (torch.cuda.get_device_name(0), os.path.basename(os.path.dirname(os.path.abspath(lib))), n / (1 << 30), args.kind))
    print("| team A (front end) | share | team B (back end) | share |")
    print("|---|---|---|---|")
    for k, (ra, rb) in enumerate(ROWS):
        print("| %s | %.1f %% | %s | %.1f %% |" % (ra, 100.0 * a[k] / max(ta, 1), rb, 100.0 * b[k] / max(tb, 1)))
    print("| team total (cycles) | %.3g | | %.3g |" % (ta, tb))


if __name__ == "__main__":
    main()
