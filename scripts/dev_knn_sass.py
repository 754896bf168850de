"""What the kNN sweep's consumer loop compiles to, without a GPU: ptxas resource usage of every knn_sweep2_kernel
instantiation and an opcode count of one steady-state step of the pipelined loop.

Compiles scanpy_b200/csrc/knn_tc2.cu alone (nvcc -gencode arch=compute_90a,code=sm_90a -Xptxas -v, the Makefile's
flags), disassembles it with cuobjdump -sass and, in the chosen instantiation (default <2, 4, false, true>: 64-proposal
lists, K = 64 pipelined loop, no stamps, integer fast path, the one bench.py runs), counts the instructions from each
`WARPGROUP.DEPBAR.LE gsb0, 0x1` (tile c's MMAs are complete, tile c+1's still run) to the next `SYNCS.PHASECHK` (the wait
for tile c+2's stage): the examination of one tile as the warpgroup executes it in the steady state.  Code the compiler
placed out of that straight line (a rare path moved behind the loop) is counted apart, as the rest of the function.

    python scripts/dev_knn_sass.py [--ng 2] [--pnks 4] [--stamps 0] [--scan int|float] [--keep DIR]

CUDA 12.9.  Every one of the 24 instantiations: 0 bytes stack frame, 0 spills, no wgmma serialisation warning (C7514 /
C7515); 168 registers for the pipelined loops (setmaxnreg), 133 to 167 for the single-buffer ones.
  <2, 4, false, false>, float max tree (--scan float): function 5192 instructions; step 1085: FMNMX 541, FSETP 132,
    FSEL 82, SEL 96, ISETP 15, BRA 19, VOTE 1, FLO 2, SHFL 36
  <2, 4, false, true>, integer max of the bit patterns:  function 5520 instructions; step 1165: VIMNMX3 30, VIMNMX 2,
    FMNMX 572, FSETP 131, FSEL 40, SEL 138, ISETP 21, BRA 25, VOTE 3, FLO 2, SHFL 36
The straight line between the two markers also holds code a tile rarely runs: the seeding at the first visit of the
sweep proper (the 36 SHFL and ~430 FMNMX of the shuffle merge), the estimate-phase max trees, the float redo of the hit
test for warps with a negative threshold (62 FMNMX, integer fast path only) and the rare path of both rows.  What a tile
without hits executes: 62 FMNMX (two rows of four quarter maxima), 2 FSETP and one VOTE with the float tree; 30 VIMNMX3
(two ternary trees), 2 VIMNMX, 4 ISETP, 1 LOP3 and one VOTE with the integer one; no MOV copies the accumulators.
"""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CSRC = os.path.join(ROOT, "scanpy_b200", "csrc")
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
SHOW = ("HGMMA", "VIMNMX3", "VIMNMX", "FMNMX", "FSETP", "FSEL", "SEL", "ISETP", "MOV", "BRA", "VOTE", "FLO", "SHFL", "CALL", "RET", "LDL", "STL")


def opcode(line):
    """'/*0af0*/  @!P0 FMNMX R3, R4, R5, !PT ;' -> 'FMNMX' (predicate and modifiers dropped)"""
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)(?:\.[A-Z0-9_.]+)?\b", line)
    return m.group(1) if m else None


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--ng", type=int, default=2, choices=(2, 4))
    p.add_argument("--pnks", type=int, default=4, choices=(0, 4, 10))
    p.add_argument("--stamps", type=int, default=0, choices=(0, 1))
    p.add_argument("--scan", default="int", choices=("int", "float"), help="fast path of the examination (SB2_KNN_SCAN)")
    p.add_argument("--keep", help="directory to keep the cubin, the ptxas log and the SASS in")
    a = p.parse_args()
    tmp = tempfile.mkdtemp(prefix="knn_sass_")
    try:
        cubin = os.path.join(tmp, "knn_tc2.cubin")
        r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-cubin",
                            "-Xptxas", "-v", "-o", cubin, os.path.join(CSRC, "knn_tc2.cu")], capture_output=True, text=True)
        if r.returncode:
            sys.exit(r.stderr)
        sass = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
        if a.keep:
            os.makedirs(a.keep, exist_ok=True)
            shutil.copy(cubin, a.keep)
            with open(os.path.join(a.keep, "ptxas.txt"), "w") as f:
                f.write(r.stderr)
            with open(os.path.join(a.keep, "sass.txt"), "w") as f:
                f.write(sass)
    finally:
        shutil.rmtree(tmp)

    # ptxas -v: registers / stack / spills per sweep instantiation
    print("ptxas -v, knn_sweep2_kernel<NG, PNKS, STAMPS, ISCAN>:")
    cur = None
    for ln in r.stderr.splitlines():
        m = re.search(r"Function properties for \S*knn_sweep2_kernelILi(\d+)ELi(\d+)ELb(\d)ELb(\d)", ln)
        if m:
            cur = f"<{m.group(1)}, {m.group(2)}, {'true' if m.group(3) == '1' else 'false'}, {'true' if m.group(4) == '1' else 'false'}>"
            continue
        if cur and "stack frame" in ln:
            print(f"  {cur:25s} {ln.strip()}", end="")
        elif cur and "Used" in ln and "registers" in ln:
            print(f"; {ln.split('ptxas info    :')[-1].strip()}")
            cur = None
    serial = [ln for ln in r.stderr.splitlines() if "serializ" in ln.lower() and "knn_sweep2" in ln]
    print(f"wgmma serialisation warnings: {len(serial)}")

    # the chosen instantiation's SASS
    iscan = int(a.scan == "int")
    name = f"knn_sweep2_kernelILi{a.ng}ELi{a.pnks}ELb{a.stamps}ELb{iscan}E"
    body, on = [], False
    for ln in sass.splitlines():
        if "Function :" in ln:
            on = name in ln
            continue
        if on:
            body.append(ln)
    ops = [(i, opcode(ln), ln) for i, ln in enumerate(body)]
    ops = [(i, op, ln) for i, op, ln in ops if op]
    total = collections.Counter(op for _, op, _ in ops)
    print(f"\n<{a.ng}, {a.pnks}, {'true' if a.stamps else 'false'}, {'true' if iscan else 'false'}>: {len(ops)} SASS instructions in the function")
    steps = []
    for j, (_, op, ln) in enumerate(ops):
        if op == "WARPGROUP" and "DEPBAR.LE gsb0, 0x1" in ln:
            for jj in range(j + 1, len(ops)):
                if ops[jj][1] == "SYNCS" and "PHASECHK" in ops[jj][2]:
                    steps.append(ops[j:jj + 1])
                    break
    if not steps:
        sys.exit("no steady-state step (WARPGROUP.DEPBAR.LE gsb0, 0x1 ... SYNCS.PHASECHK) found")
    for n, st in enumerate(steps):
        c = collections.Counter(op for _, op, _ in st)
        print(f"steady-state step {n}: {len(st)} instructions; " + ", ".join(f"{k} {c[k]}" for k in SHOW if c[k]))
    # the step the loop runs most: the longest one inside the unrolled pair (epilogue copies are shorter or equal)
    st = steps[0]
    c = collections.Counter(op for _, op, _ in st)
    print("\nopcodes of step 0, most frequent first:")
    print("  " + ", ".join(f"{k} {v}" for k, v in c.most_common()))
    print("\nwhole function: " + ", ".join(f"{k} {total[k]}" for k in SHOW if total[k]))


if __name__ == "__main__":
    main()
