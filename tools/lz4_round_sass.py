"""Static check of the candidate rounds' machine code (no GPU needed).

    python tools/lz4_round_sass.py [--csrc DIR]

Cross-compiles lz4_kernels.cu for sm_90a, finds the candidate round (lz_candidates in lz4_pipe.cuh) in both kernels that
run it, lz4_blocks_pipe_kernel and zstd_blocks_kernel, and reports per round: instructions, branch instructions
(BRA / BSSY / BSYNC / BREAK), how many of the eight verifying LDS are issued before the first instruction that reads
one of their results, and the kernel's registers, spill bytes and named barriers.  The round is the loop whose body holds the first hash multiply
(x * 2654435761 >> 20); its first LDS after that multiply is the first table read, its STS.64 the store of the offsets.

Exits 1 if a BRA or BSSY lies between the first table LDS and that STS.64 in either kernel: the round body is meant to be
straight-line code there (DESIGN.md §3.4).
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = {"lz4_blocks_pipe_kernel": "_Z22lz4_blocks_pipe_kernel", "zstd_blocks_kernel": "_Z18zstd_blocks_kernel"}
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
BRANCHES = ("BRA", "BSSY", "BSYNC", "BREAK")


def compile_cubin(csrc, tmp):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    cubin = os.path.join(tmp, "lz4_kernels.cubin")
    r = subprocess.run([nvcc, "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-o", cubin, os.path.join(csrc, "lz4_kernels.cu")], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise SystemExit("nvcc failed")
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.dirname(nvcc) else "cuobjdump", "-sass", cubin],
                          capture_output=True, text=True, check=True).stdout
    return sass, r.stdout + r.stderr


def ptxas_info(log, mangled):
    """registers, spill bytes (stores + loads), named barriers of one kernel from the -Xptxas -v log"""
    lines = log.splitlines()
    for j, ln in enumerate(lines):
        if "Compiling entry function '%s" % mangled in ln:
            blk = "\n".join(lines[j:j + 4])
            regs = int(re.search(r"Used (\d+) registers", blk).group(1))
            bars = int(re.search(r"used (\d+) barriers", blk).group(1))
            sp = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
            return regs, int(sp.group(1)) + int(sp.group(2)), bars
    raise SystemExit("ptxas log has no entry for %s" % mangled)


def function_insns(sass, mangled):
    """[(address, text)] of one kernel"""
    out, on = [], False
    for ln in sass.splitlines():
        if "Function : " in ln:
            on = ln.split("Function : ")[1].strip().startswith(mangled)
            continue
        m = INSN.search(ln) if on else None
        if m:
            out.append((int(m.group(1), 16), m.group(2)))
    return out


def opcode(text):
    t = re.sub(r"^@!?U?P\w+\s+", "", text)
    return t.split()[0] if t else ""


def operands(text):
    t = re.sub(r"^@!?U?P\w+\s+", "", text)
    parts = t.split(None, 1)
    return [x.strip() for x in parts[1].split(",")] if len(parts) > 1 else []


def regs_in(ops):
    return set(int(x) for op in ops for x in re.findall(r"\bR(\d+)\b", op))


def analyse(insns):
    # the hash multiply: IMAD by 0x9e3779b1 whose result is shifted right by 20 within a few instructions
    anchor = None
    for j, (_, t) in enumerate(insns):
        if opcode(t).startswith("IMAD") and "-0x61c8864f" in t:
            d = operands(t)[0]
            if any(re.match(r"SHF\.R\.U32\.HI %s, RZ, 0x14, %s$" % (d, d), insns[k][1]) for k in range(j + 1, min(j + 8, len(insns)))):
                anchor = j
                break
    if anchor is None:
        raise SystemExit("no hash multiply found")
    a_addr = insns[anchor][0]
    # the round loop: the first backward branch after the multiply that jumps to or before it
    back = None
    for j in range(anchor + 1, len(insns)):
        t = insns[j][1]
        if opcode(t).startswith("BRA"):
            m = re.search(r"0x([0-9a-f]+)\s*$", t)
            if m and int(m.group(1), 16) <= a_addr:
                back, start_addr = j, int(m.group(1), 16)
                break
    if back is None:
        raise SystemExit("no round loop found")
    start = next(j for j, (a, _) in enumerate(insns) if a == start_addr)
    body = insns[start:back + 1]
    n_branch = sum(opcode(t).split(".")[0] in BRANCHES for _, t in body)
    first_lds = next(j for j in range(anchor, back) if opcode(insns[j][1]) == "LDS")
    sts = next(j for j in range(anchor, back) if opcode(insns[j][1]) == "STS.64")
    window = insns[first_lds:sts + 1]
    bad = [(a, t) for a, t in window if opcode(t).split(".")[0] in ("BRA", "BSSY")]
    lds = [j for j in range(first_lds, sts) if opcode(insns[j][1]) == "LDS"]
    # verifying LDS issued before the first instruction that reads one of their results
    verify, before, dst = lds[4:12], 0, set()
    for j in range(verify[0] if verify else sts, sts):
        op, ops = opcode(insns[j][1]), operands(insns[j][1])
        srcs = ops if op.startswith(("ST", "RED", "ATOM")) else ops[1:]
        if regs_in(srcs) & dst:
            break
        if j in verify:
            dst |= regs_in(ops[:1])
            before += 1
    return dict(insns=len(body), branches=n_branch, lds=len(lds), before=before, nverify=len(verify), bad=bad)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--csrc", default=os.path.join(ROOT, "zstdmt_b200", "csrc"), help="source directory holding lz4_kernels.cu")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        sass, log = compile_cubin(args.csrc, tmp)
    ok = True
    for name, mangled in KERNELS.items():
        regs, spill, bars = ptxas_info(log, mangled)
        r = analyse(function_insns(sass, mangled))
        print("%-24s instructions/round %4d  branches/round %3d  LDS table..STS.64 %2d  verify LDS before first use %d/%d  "
              "BRA/BSSY table..STS.64: %d  | %d registers, %d spill bytes, %d barriers"
              % (name, r["insns"], r["branches"], r["lds"], r["before"], r["nverify"], len(r["bad"]), regs, spill, bars))
        for a, t in r["bad"]:
            print("    /*%04x*/ %s" % (a, t))
        ok &= not r["bad"]
    print("PASS" if ok else "FAIL: the candidate round branches between its first table read and the offset store")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
