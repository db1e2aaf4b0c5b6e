#!/usr/bin/env python3
"""Instruction mix of the Riccati kernel (K3, mpc_riccati_kernel) per region of its node loops, from the compiler's output; no GPU needed.

  python tools/sass_regions.py                 # the working tree
  python tools/sass_regions.py --rev HEAD~1    # another commit, side by side with the working tree

Compiles kernels/mpc_kernels.cu for sm_90a with -lineinfo (the library's flags), disassembles K3 with nvdisasm's inline line information and
attributes every instruction to the kernel source line it was inlined into. The regions are the spans between the sweep's barriers, found by
anchor lines in the kernel source: the prologue, the loop top with the event-node path, phases 1 and 2, the factorisation branch and the helper
branch of phase 3, phase 4 with the expand() that rebuilds the next node, and the forward rollout. Counts are static (instructions in the binary),
not issued instructions.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
SRC = "qm_control_b200/csrc/kernels/mpc_kernels.cu"
KERNEL = "mpc_riccati_kernel"
# (region, regular expression of the first kernel source line of the region); a line belongs to the last region whose anchor precedes it
ANCHORS = [
    ("prologue", r"mpc_riccati_kernel\("),
    ("loop top, event node", r"for \(int k = N - 1; k >= 0; --k\)"),
    ("phase 1", r"gAB\.wait\(\); if \(QMB_TMA\) __syncthreads\(\);"),
    ("phase 2", r"// ---- phase 2:"),
    ("phase 3 factorisation", r"issue_q\(k\);"),
    ("phase 3 helpers", r"if \(QMB_TMA\) gQ\.wait\(\);"),
    ("phase 4 + expand()", r"if \(sm\.flag\) \{ st \|= MST_NOT_PD"),
    ("rollout", r"// ---- forward rollout"),
    ("epilogue", r"armijo = warp_sum\(armijo\)"),
]
SWEEP = ("loop top, event node", "phase 1", "phase 2", "phase 3 factorisation", "phase 3 helpers", "phase 4 + expand()")
CLASSES = ("fp64", "dmma", "int", "move", "ctrl", "shfl", "lds", "sts", "mem", "other")


def op_class(op):
    base = op.split(".")[0]
    if base == "DMMA":
        return "dmma"
    if base in ("DFMA", "DADD", "DMUL", "DSETP", "DMNMX") or op.startswith("MUFU.RSQ64") or op.startswith("MUFU.RCP64"):
        return "fp64"
    if base == "SHFL":
        return "shfl"
    if base == "LDS" or base == "LDSM":
        return "lds"
    if base == "STS":
        return "sts"
    if base in ("MOV", "UMOV", "SEL", "FSEL", "USEL", "CS2R", "S2R", "S2UR", "R2UR", "MOV64") or op.startswith("IMAD.MOV") or op.startswith("IMAD.U32"):
        return "move"
    if base in ("BRA", "BRX", "JMP", "BSSY", "BSYNC", "EXIT", "CALL", "RET", "WARPSYNC", "BAR", "NOP", "YIELD", "BPT", "VOTE", "VOTEU", "MEMBAR", "ELECT", "ACQBULK", "DEPBAR", "ERRBAR"):
        return "ctrl"
    if base in ("LDG", "STG", "LDL", "STL", "LD", "ST", "LDC", "ULDC", "ATOM", "ATOMG", "ATOMS", "RED", "REDG", "SYNCS", "UBLKCP", "LDGSTS", "LDGDEPBAR", "UBLKPF", "CCTL", "FENCE"):
        return "mem"
    if base in ("IMAD", "IADD3", "VIADD", "ISETP", "LEA", "LOP3", "SHF", "IMNMX", "VIMNMX", "IABS", "POPC", "FLO", "BMSK", "SGXT", "PRMT", "PLOP3", "P2R", "R2P", "IMUL", "I2F", "F2I", "LEA", "UIADD3", "UIMAD", "ULEA",
                "ULOP3", "USHF", "UISETP", "UPRMT", "UFLO", "UPOPC", "UBMSK", "USGXT", "UPLOP3", "ISCADD", "IDP", "I2IP", "UP2UR", "UR2UP"):
        return "int"
    return "other"


def anchor_lines(src_text):
    lines = src_text.splitlines(); start = None; out = []
    for name, rx in ANCHORS:
        pat = re.compile(rx)
        for i in range(0 if start is None else start, len(lines)):
            if pat.search(lines[i]):
                out.append((i + 1, name)); start = i; break
        else:
            sys.exit("anchor of region %r not found in %s" % (name, SRC))
    return out


def compile_and_count(tree, tmp, tag):
    src = os.path.join(tree, SRC); cubin = os.path.join(tmp, tag + ".cubin")
    cmd = [os.path.join(CUDA, "bin", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-cubin", "-o", cubin, src]
    r = subprocess.run(cmd, cwd=os.path.dirname(src), capture_output=True, text=True)
    if r.returncode:
        sys.exit(r.stderr)
    ptxas = [l.strip() for l in r.stderr.splitlines()]
    info = ""
    for i, l in enumerate(ptxas):
        if "Function properties for" in l and KERNEL in l:
            info = "; ".join(ptxas[i + 1:i + 3])
    sass = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "-c", "-gi", cubin], capture_output=True, text=True, check=True).stdout
    anchors = anchor_lines(open(src).read()); fname = os.path.basename(SRC)
    counts = collections.OrderedDict((name, collections.Counter()) for _, name in anchors)
    inside = False; region = anchors[0][1]; nbar = collections.Counter()
    for line in sass.splitlines():
        s = line.strip()
        if s.startswith(".text."):
            inside = KERNEL in s; continue
        if not inside:
            continue
        if s.startswith("//## File"):
            # an inlined chain is printed one hop per comment, the last comment naming a line of the kernel body; hops inside helper functions
            # (above the kernel) and inside other files leave the region as it is
            locs = re.findall(r'"([^"]+)", line (\d+)', s)
            own = [int(n) for f, n in locs if os.path.basename(f) == fname]
            if own and own[-1] >= anchors[0][0]:
                for a, name in anchors:
                    if own[-1] >= a:
                        region = name
            continue
        m = re.match(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", s)
        if not m:
            continue
        op = m.group(1); counts[region][op_class(op)] += 1; counts[region]["total"] += 1
        if op.startswith("BAR.SYNC") or op.startswith("BAR.RED") or op.startswith("BAR.ARV"):
            nbar[region] += 1
    return counts, info, nbar


def table(counts):
    rows = []
    for name, c in counts.items():
        rows.append([name, c["total"], c["total"] - c["fp64"] - c["dmma"]] + [c[k] for k in CLASSES])
    sweep = [r for r in rows if r[0] in SWEEP]
    rows.append(["sweep (node loop)"] + [sum(r[i] for r in sweep) for i in range(1, len(rows[0]))])
    rows.append(["kernel"] + [sum(r[i] for r in rows[:len(counts)]) for i in range(1, len(rows[0]))])
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rev", help="also count this git revision's kernel and print the difference")
    args = ap.parse_args()
    hdr = ["region", "total", "non-fp64"] + list(CLASSES)
    with tempfile.TemporaryDirectory() as tmp:
        trees = [("working tree", ROOT)]
        if args.rev:
            t = os.path.join(tmp, "rev"); os.makedirs(t)
            arch = subprocess.run(["git", "-C", ROOT, "archive", args.rev, "qm_control_b200/csrc", "include"], capture_output=True, check=True).stdout
            subprocess.run(["tar", "-x", "-C", t], input=arch, check=True)
            trees.insert(0, (args.rev, t))
        results = []
        for i, (tag, tree) in enumerate(trees):
            counts, info, nbar = compile_and_count(tree, tmp, "t%d" % i)
            results.append(table(counts))
            print("== %s: %s  (ptxas: %s; CTA barriers per region: %s)" % (KERNEL, tag, info, ", ".join("%s %d" % kv for kv in nbar.items())))
            w = [max(len(hdr[0]), max(len(r[0]) for r in results[-1]))] + [max(6, len(h)) for h in hdr[1:]]
            print("  ".join(h.ljust(w[0]) if j == 0 else h.rjust(w[j]) for j, h in enumerate(hdr)))
            for r in results[-1]:
                print("  ".join(str(v).ljust(w[0]) if j == 0 else str(v).rjust(w[j]) for j, v in enumerate(r)))
            print()
        if len(results) == 2:
            print("== change, %s -> working tree (total / non-fp64)" % args.rev)
            for a, b in zip(*results):
                print("  %-24s %6d -> %6d (%+5d)   %6d -> %6d (%+5d)" % (a[0], a[1], b[1], b[1] - a[1], a[2], b[2], b[2] - a[2]))


if __name__ == "__main__":
    main()
