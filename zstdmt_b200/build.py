"""Build the in-tree native libraries (no torch extension machinery, plain nvcc / gcc).

  zstdmt_b200/libzstdmt_b200.so   CUDA kernels (sm_90a) + host pipeline + C-ABI   [the product]
  zstdmt_b200/libzmt_datagen.so   synthetic input generator (harness/datagen.c)     [bench / test harness, no dependencies]
  zstdmt_b200/libzmt_memio.so     in-memory fn_read / fn_write drivers of the C-ABI [bench / test harness, links the product]
  zstdmt_b200/libzlazy_dict_twin.so  CPU twin of the zstd search class against a dictionary   [test infrastructure]
  oracle/liboracle.so             CPU restatement                                  [test infrastructure]
  oracle/libchain_twin.so         CPU twin of the chain-search encoders            [test infrastructure]
  oracle/libzlazy_twin.so,        links to libchain_twin.so under the per-class names that test trees and tools
  oracle/liblz4hc_twin.so           load the zstd level 6-12 and LZ4 level 10-12 twins by
  oracle/_ref/libzstdmt_ref.so    unmodified reference wrapper, only where the reference tree exists (oracle/Makefile REF)
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libzstdmt_b200.so")
HSRC = os.path.join(HERE, "harness")
LIB_GEN = os.path.join(HERE, "libzmt_datagen.so")
LIB_MEMIO = os.path.join(HERE, "libzmt_memio.so")
LIB_DICT_TWIN = os.path.join(HERE, "libzlazy_dict_twin.so")
LIB_TWIN = os.path.join(ROOT, "oracle", "libchain_twin.so")
LIB_TWIN_NAMES = [os.path.join(ROOT, "oracle", f) for f in ("libzlazy_twin.so", "liblz4hc_twin.so")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-pthread", "-shared",
]


def _sources():
    srcs = []
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cpp", ".c")):
            srcs.append(os.path.join(CSRC, f))
    return srcs


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_product(force=False, verbose=False, defines=(), out_dir=None):
    """The product library; with `defines` (e.g. ["ZMT_PHASE_PROBE"]) an instrumented variant, built as
    out_dir/libzstdmt_b200.so (out_dir is required then, so a variant never replaces the product)."""
    if defines and not out_dir:
        raise ValueError("a library built with extra defines goes to its own out_dir")
    lib = os.path.join(out_dir, "libzstdmt_b200.so") if out_dir else LIB
    srcs = _sources()
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    if not force and not _stale(lib, deps):
        return lib
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    tmp = lib + ".tmp.%d" % os.getpid()         # link under a scratch name, then rename: readers never see a half-written library
    cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + srcs + ["-lpthread"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed building libzstdmt_b200.so")
    os.replace(tmp, lib)
    return lib


def build_harness(force=False):
    """The harness libraries (plain gcc).  libzmt_memio.so resolves LZ4MT_* / ZSTDCB_* from the product library."""
    gen_src, io_src = os.path.join(HSRC, "datagen.c"), os.path.join(HSRC, "memio_glue.c")
    if force or _stale(LIB_GEN, [gen_src]):
        r = subprocess.run(["gcc", "-O3", "-fPIC", "-pthread", "-shared", "-o", LIB_GEN, gen_src, "-lpthread"], cwd=ROOT, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr); raise RuntimeError("gcc failed building libzmt_datagen.so")
    if force or _stale(LIB_MEMIO, [io_src, LIB]):
        r = subprocess.run(["gcc", "-O3", "-fPIC", "-shared", "-DGLUE_PREFIX=zmt_", "-o", LIB_MEMIO, io_src, "-L" + HERE, "-l:libzstdmt_b200.so",
                            "-Wl,-rpath,$ORIGIN"], cwd=ROOT, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr); raise RuntimeError("gcc failed building libzmt_memio.so")
    # CPU twin of the zstd search class against a dictionary (shares zstd_lazy_rule.h with the kernels)
    tw_src = os.path.join(HSRC, "zlazy_dict_twin.c")
    if force or _stale(LIB_DICT_TWIN, [tw_src, os.path.join(CSRC, "zstd_lazy_rule.h")]):
        r = subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-o", LIB_DICT_TWIN, tw_src], cwd=ROOT, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr); raise RuntimeError("gcc failed building libzlazy_dict_twin.so")


def build_oracle(force=False):
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("oracle build failed")
    # CPU twin of the zstd level 6-12 and LZ4 level 10-12 classes (shares their rule headers with the kernels)
    src, rules = os.path.join(ROOT, "oracle", "chain_twin.c"), [os.path.join(CSRC, f) for f in ("lz4_hc_rule.h", "zstd_lazy_rule.h")]
    if force or _stale(LIB_TWIN, [src] + rules):
        r = subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-o", LIB_TWIN, src], cwd=ROOT, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr); raise RuntimeError("gcc failed building oracle/libchain_twin.so")
    for name in LIB_TWIN_NAMES:
        target = os.path.basename(LIB_TWIN)
        if not (os.path.islink(name) and os.readlink(name) == target):
            tmp = name + ".tmp.%d" % os.getpid()
            os.symlink(target, tmp)
            os.replace(tmp, name)


def build_cli():
    """Reference CLI (unmodified programs/main.c) linked against the product library — only where the reference tree exists."""
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "cli"], capture_output=True, text=True)


def build_all(force=False, verbose=False):
    build_product(force=force, verbose=verbose)
    build_harness(force=force)
    build_oracle(force=force)
    build_cli()


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("ok:", LIB)
