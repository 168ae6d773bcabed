#!/usr/bin/env python3
"""Instructions per trellis step of the Viterbi forward pass, from the sm_90a SASS (no GPU needed).

Compiles welle.io_b200/csrc/viterbi.cu for sm_90a with the flags of the library's Makefile, finds in each viterbi_kernel
instance the group loop (the innermost loop that holds the packed add-compare-select minima: six trellis steps per
iteration) and prints its instructions per step, split by the pipe that executes them, with the registers and spills
ptxas reports for the kernel.

Pipes (sm_90, 16 lanes per scheduler per clock each): "alu" = integer ALU (IADD3, LOP3, PRMT, VIMNMX, ...), "fma" = the
FMA pipe's integer forms (IMAD and its IADD / MOV / SHL aliases, IDP.4A); everything else (memory, uniform datapath,
control, MOV) is listed apart.

    python scripts/vit_sass_count.py [--keep DIR] [--nvcc PATH]
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "welle.io_b200", "csrc")
STEPS_PER_ITER = 6

ALU = {"IADD3", "LOP3", "PRMT", "VIMNMX", "VIMNMX3", "VIADDMNMX", "VIADD", "SHF", "LEA", "ISETP", "SEL", "IMNMX",
       "P2R", "R2P", "PLOP3", "IABS", "BMSK", "SGXT", "FLO", "POPC", "BREV", "ICMP", "FSEL", "FMNMX", "FSETP"}
FMA = {"IMAD", "IDP", "IMUL", "FFMA", "FMUL", "FADD"}
PACKED_MIN = re.compile(r"^(VIMNMX|VIMNMX3|VIADDMNMX)\.S16x2")
LINE = re.compile(r"^\s+/\*([0-9a-f]{4,})\*/\s+(@!?U?P[0-9T]\s+)?([A-Z0-9_.][A-Za-z0-9_.]*)(.*?);")


def pipe_of(op):
    base = op.split(".")[0]
    if base in FMA:
        return "fma"
    if base in ALU:
        return "alu"
    if base.startswith(("LD", "ST", "ATOM", "RED", "CCTL", "SYNCS", "UBLKCP")):
        return "mem"
    if base.startswith("U") or base in ("S2UR", "R2UR"):
        return "uniform"
    return "other"


def functions(sass):
    """{mangled name: [(address, opcode, operands)]}"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = LINE.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(3), m.group(4)))
    return out


def group_loop(code):
    """The innermost backward-branch range that holds the kernel's packed minima."""
    best = None
    for addr, op, args in code:
        if not op.startswith("BRA"):
            continue
        m = re.search(r"0x([0-9a-f]+)", args)
        if not m or int(m.group(1), 16) >= addr:
            continue
        lo = int(m.group(1), 16)
        body = [(a, o) for a, o, _ in code if lo <= a <= addr]
        mins = sum(1 for _, o in body if PACKED_MIN.match(o))
        if mins < 16 * STEPS_PER_ITER:
            continue
        if best is None or len(body) < len(best):
            best = body
    return best


def ptxas_usage(log):
    """{mangled name: (registers, spill stores, spill loads)}"""
    out, name, spills = {}, None, (0, 0)
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spills = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            out[name] = (int(m.group(1)),) + spills
            name = None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--nvcc", default=os.environ.get("NVCC", "nvcc"))
    ap.add_argument("--keep", help="directory for the object, the SASS and the ptxas log (default: a temporary one)")
    a = ap.parse_args()
    work = a.keep or tempfile.mkdtemp(prefix="vit_sass_")
    os.makedirs(work, exist_ok=True)
    obj = os.path.join(work, "viterbi.o")
    cmd = [a.nvcc, "-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
           "-Xcompiler", "-fPIC,-ffp-contract=off", "-Xptxas", "-v", "-c", os.path.join(CSRC, "viterbi.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        return 1
    usage = ptxas_usage(r.stderr)
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    if a.keep:
        with open(os.path.join(work, "viterbi.sass"), "w") as f:
            f.write(sass)
        with open(os.path.join(work, "ptxas.log"), "w") as f:
            f.write(r.stderr)
    found = 0
    for name, code in sorted(functions(sass).items()):
        if "viterbi_kernel" not in name:
            continue
        inst = "viterbi_kernel<" + ("true" if "ILb1E" in name else "false") + ">"
        body = group_loop(code)
        if body is None:
            print(f"{inst}: no group loop found")
            continue
        found += 1
        ops = collections.Counter(o for _, o in body)
        pipes = collections.Counter()
        for o, n in ops.items():
            pipes[pipe_of(o)] += n
        regs, sst, sld = usage.get(name, (0, 0, 0))
        n = len(body)
        print(f"{inst}: {regs} registers, {sst} B spill stores, {sld} B spill loads; group loop {n} instructions "
              f"= {n / STEPS_PER_ITER:.1f} per trellis step")
        for p in ("alu", "fma", "mem", "uniform", "other"):
            if not pipes[p]:
                continue
            mix = sorted(((c, o) for o, c in ops.items() if pipe_of(o) == p), reverse=True)
            desc = ", ".join(f"{o} {c / STEPS_PER_ITER:.1f}" for c, o in mix[:8])
            print(f"  {p:8s} {pipes[p] / STEPS_PER_ITER:6.1f} per step  ({desc})")
    return 0 if found == 2 else 1


if __name__ == "__main__":
    sys.exit(main())
