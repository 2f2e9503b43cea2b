#!/usr/bin/env python3
"""Opcode census of the scan kernels' scoring loops, read from the sm_90a SASS (no GPU needed).

Compiles torchpq_b200/csrc/scan.cu with the Makefile's flags into a temporary directory (or reads --obj), disassembles
the cell-major kernel and the query-major kernel with cuobjdump, splits each into basic blocks and reports every block
that holds at least --min-lookups 4-byte LDS: one LDS is one LUT lookup, so instructions / LDS is the issue cost of a
lookup.  The ideal is 3 (PRMT + LDS + FADD).

    python scripts/sass_census.py                 # compile scan.cu, census both kernels
    python scripts/sass_census.py --obj scan.o    # census an existing object
"""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "torchpq_b200", "csrc")
KERNELS = {
    "cell": "_ZN3tpq22ivfpq_cell_scan_kernelILi12ELi7EEEvNS_8CellArgsE",
    "query-major": "_ZN3tpq17ivfpq_scan_kernelILi64ELi8ELi2ELi0ELb0EEEvNS_8ScanArgsENS_8ScanSmemE",
}
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
TARGET = re.compile(r"(0x[0-9a-f]+)\s*$")
ENDS_BLOCK = ("BRA", "BRX", "JMP", "JMX", "CALL", "RET", "EXIT", "BSSY", "BSYNC", "BREAK", "WARPSYNC")


def nvcc():
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    for p in (shutil.which("nvcc"), os.path.join(cuda, "bin", "nvcc")):
        if p and os.path.exists(p):
            return p
    sys.exit("nvcc not found (set CUDA_HOME)")


def compile_scan(out_dir):
    obj = os.path.join(out_dir, "scan.o")
    cmd = [nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
           "--expt-relaxed-constexpr", "-c", os.path.join(CSRC, "scan.cu"), "-o", obj]
    subprocess.run(cmd, check=True, cwd=CSRC, stderr=subprocess.DEVNULL)
    return obj


def disassemble(obj, fun):
    cuobjdump = os.path.join(os.path.dirname(nvcc()), "cuobjdump")
    txt = subprocess.run([cuobjdump, "-sass", "-fun", fun, obj], check=True, capture_output=True, text=True).stdout
    insns = []
    for line in txt.splitlines():
        m = INSN.match(line)
        if m:
            insns.append((int(m.group(1), 16), m.group(2)))
    if not insns:
        sys.exit(f"{fun}: not found in {obj}")
    return insns


def opcode(text):
    tok = text.split()
    return tok[1] if tok[0].startswith("@") else tok[0]


def basic_blocks(insns):
    leaders = {insns[0][0]}
    for i, (addr, text) in enumerate(insns):
        op = opcode(text).split(".")[0]
        if op in ENDS_BLOCK:
            m = TARGET.search(text)
            if m:
                leaders.add(int(m.group(1), 16))
            if i + 1 < len(insns):
                leaders.add(insns[i + 1][0])
    blocks, cur = [], []
    for addr, text in insns:
        if addr in leaders and cur:
            blocks.append(cur)
            cur = []
        cur.append((addr, text))
    blocks.append(cur)
    return blocks


def census(name, insns, min_lookups):
    print(f"{name}: {len(insns)} instructions ({len(insns) * 16 / 1024:.1f} KB of code)")
    tot_n, tot_l, tot_ops = 0, 0, collections.Counter()
    for blk in basic_blocks(insns):
        ops = collections.Counter(opcode(t) for _, t in blk)
        lookups = ops["LDS"]
        if lookups < min_lookups:
            continue
        tot_n += len(blk)
        tot_l += lookups
        tot_ops.update(ops)
        top = ", ".join(f"{o} {c}" for o, c in ops.most_common(10))
        print(f"  block @0x{blk[0][0]:05x}: {len(blk):5d} insns, {lookups:4d} lookups, {len(blk) / lookups:.2f} per lookup"
              f"  [{top}]")
    if tot_l:
        print(f"  scoring blocks together: {tot_n} insns / {tot_l} lookups = {tot_n / tot_l:.2f} per lookup")
        print("  " + ", ".join(f"{o} {c}" for o, c in tot_ops.most_common()))
    else:
        print("  no scoring block found")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--obj", help="object or cubin to read instead of compiling scan.cu")
    ap.add_argument("--min-lookups", type=int, default=32, help="LDS count that makes a basic block a scoring block")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        obj = args.obj or compile_scan(tmp)
        for name, fun in KERNELS.items():
            census(name, disassemble(obj, fun), args.min_lookups)


if __name__ == "__main__":
    main()
