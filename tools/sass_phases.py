"""SASS of the fused field kernel's consumer phases, without a GPU.  Compiles one instantiation of k_field_tc with the flags of
sdfstudio_b200/build.py, disassembles it with its inline line info and attributes every instruction to the call in the kernel body
it was inlined from.  For each phase function called from the kernel body (epi_e0, epi_e1, epi_eb1, epi_eb0, colour_copy, epi_ec0,
epi_ec1; one row per call site) it prints the instruction count, the main opcodes, and how many of the phase's loads are issued
directly behind one of its stores, i.e. the loads whose preceding instruction in the phase is a store, and in how many batches its
loads are issued (runs of loads with no store of the phase between them).  A load placed behind a store waits for whatever the
store was waiting for, so a phase whose per-element loads all sit behind the previous element's store runs its elements one after
another.

    usage: tools/sass_phases.py [p2_torch | p2_tcnn | p1_torch | p1_tcnn] [--keep DIR]"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sdfstudio_b200 import build as b  # noqa: E402

KERNEL_SRC = os.path.join(b.CSRC, "field_tc_kernel.cuh")
NVDISASM = os.path.join(os.path.dirname(b.NVCC), "nvdisasm")
LOADS = {"LDS", "LDG", "LD", "LDL", "LDSM"}
STORES = {"STS", "STG", "ST", "STL"}
SHOWN = ["LDS", "LDG", "STS", "STG", "FADD", "FMUL", "FFMA", "MUFU", "F2FP", "PRMT", "IMAD", "SHFL"]


def phase_calls():
    """{line number in field_tc_kernel.cuh: phase function} for the phase calls inside the body of k_field_tc"""
    lines = open(KERNEL_SRC).read().split("\n")
    start = next(i for i, ln in enumerate(lines) if re.search(r"__global__ .*\bk_field_tc\(", ln))
    calls = {}
    for i in range(start, len(lines)):
        m = re.search(r"\b(epi_\w+|colour_copy)\s*(<[^>()]*>)?\s*\(", lines[i])
        if m:
            calls[i + 1] = m.group(1)
    return calls


def compile_cubin(inst, outdir):
    src = os.path.join(b.CSRC, f"field_tc_{inst}.cu")
    cubin = os.path.join(outdir, f"field_tc_{inst}.cubin")
    r = subprocess.run([b.NVCC, *b.FLAGS, "-cubin", src, "-o", cubin], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}{r.stderr}")
    log = (r.stdout + r.stderr).split("\n")
    ptxas = []
    for i, ln in enumerate(log):     # ptxas -v lines of the k_field_tc entry
        if "Compiling entry function" in ln and "k_field_tc" in ln:
            ptxas = [s.strip() for s in log[i + 1:i + 3] if s.strip()]
    return cubin, ptxas


def disassemble(cubin):
    """[(opcode, outermost kernel-body line)] of k_field_tc in address order"""
    out = subprocess.run([NVDISASM, "-gi", "-c", cubin], capture_output=True, text=True, check=True).stdout
    kname = os.path.basename(KERNEL_SRC)
    insts, in_kernel, body_line, pending = [], False, None, []
    for ln in out.split("\n"):
        s = ln.strip()
        if s.startswith(".text."):
            in_kernel = "k_field_tc" in s
            continue
        if not in_kernel:
            continue
        if s.startswith("//##"):
            pending.append(s)
            continue
        if pending:     # a new chain: innermost frame first, the kernel body's own line last
            m = re.search(r'File "([^"]*)", line (\d+)$', pending[-1])
            body_line = int(m.group(2)) if m and os.path.basename(m.group(1)) == kname else None
            pending = []
        m = re.match(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", s)
        if m:
            insts.append((m.group(1).split(".")[0], body_line))
    return insts


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("inst", nargs="?", default="p2_torch", choices=["p2_torch", "p2_tcnn", "p1_torch", "p1_tcnn"])
    ap.add_argument("--keep", default=None, help="directory for the cubin (default: a temporary one)")
    args = ap.parse_args()
    calls = phase_calls()
    with tempfile.TemporaryDirectory() as tmp:
        outdir = args.keep or tmp
        os.makedirs(outdir, exist_ok=True)
        cubin, ptxas = compile_cubin(args.inst, outdir)
        insts = disassemble(cubin)
    print(f"k_field_tc, field_tc_{args.inst}.cu: {len(insts)} instructions")
    for s in ptxas:
        print(f"  ptxas: {s}")
    rows = collections.OrderedDict((ln, {"ops": collections.Counter(), "loads": 0, "behind": 0, "batches": 0}) for ln in sorted(calls))
    prev, prev_mem = {}, {}
    for op, ln in insts:
        if ln not in rows:
            continue
        r = rows[ln]
        r["ops"][op] += 1
        if op in LOADS:
            r["loads"] += 1
            if prev.get(ln) in STORES:
                r["behind"] += 1
            if prev_mem.get(ln) not in LOADS:
                r["batches"] += 1
        if op in LOADS or op in STORES:
            prev_mem[ln] = op
        prev[ln] = op
    print(f"{'phase (kernel line)':<22}{'instr':>7}{'loads':>7}{'behind a store':>16}{'load batches':>14}   " + " ".join(f"{o:>5}" for o in SHOWN))
    for ln, r in rows.items():
        n = sum(r["ops"].values())
        if n == 0:
            continue
        print(f"{calls[ln] + ' (' + str(ln) + ')':<22}{n:>7}{r['loads']:>7}{r['behind']:>16}{r['batches']:>14}   " + " ".join(f"{r['ops'][o]:>5}" for o in SHOWN))


if __name__ == "__main__":
    main()
