#!/usr/bin/env python
"""regenerate profiles/r02_sass_evidence.txt (static SASS mnemonic counts per kernel) and profiles/r02_ptxas_resources.txt
(registers / spills / static shared memory from csrc/build/*.ptxas.log) for the library as built."""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "spark-network-traffic-classifier_b200", "b200flow", "libb200flow.so")
BUILD = os.path.join(ROOT, "spark-network-traffic-classifier_b200", "csrc", "build")
KEEP_ROUTE = {"<7, 8, 2, 2>", "<7, 16, 1, 2>", "<9, 32, 1, 2>", "<9, 8, 2, 2>", "<7, 8, 2, 1>", "<0, 8, 2, 0>"}
COLS = ["UBLKCP", "SYNCS", "LDGSTS", "REDUX", "ATOMS", "ATOMG", "REDG", "MATCH", "VOTE", "SHFL", "DFMA", "DMUL", "MUFU.RCP64H", "LDS", "STS", "BAR.SYNC", ".EF"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    clean = []
    for n in out:
        n = re.sub(r"^void ", "", n)
        n = re.sub(r"\(.*$", "", n).replace("b200flow::", "")
        clean.append(n)
    return clean


def keep(name):
    if name.startswith("route_hist_level_kernel"):
        return any(name.endswith(k) for k in KEEP_ROUTE)
    return True


def sass():
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    funcs, cur = collections.OrderedDict(), None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); funcs[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur:
            funcs[cur].append(m.group(1))
    names = demangle(list(funcs))
    lines = []
    for (mangled, ins), name in zip(funcs.items(), names):
        if not keep(name):
            continue
        row = [name, str(len(ins))]
        for c in COLS:
            if c == ".EF":
                row.append(str(sum(1 for i in ins if ".EF" in i.split()[0] or (i.startswith("@") and ".EF" in i.split()[1]))))
            else:
                row.append(str(sum(1 for i in ins if re.search(r"(^|\s)" + re.escape(c) + r"(\.|\s|$)", " ".join(i.split()[:2])))))
        lines.append(" | ".join(row))
    return lines


def ptxas():
    rows = []
    for f in sorted(os.listdir(BUILD)):
        if not f.endswith(".ptxas.log"):
            continue
        txt = open(os.path.join(BUILD, f)).read()
        for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                             r"ptxas info\s+: Used (\d+) registers(?:, used \d+ barriers)?(?:, (\d+) bytes smem)?", txt):
            rows.append((m.group(1), m.group(5), m.group(3), m.group(4), m.group(6) or "0"))
    names = demangle([r[0] for r in rows])
    return [" | ".join((n,) + r[1:]) for n, r in zip(names, rows) if keep(n)]


if __name__ == "__main__":
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    with open(os.path.join(ROOT, "profiles", "r02_sass_evidence.txt"), "w") as f:
        f.write("# SASS evidence (cuobjdump -sass libb200flow.so, sm_90a): static instruction counts per kernel for the mnemonics that matter (tools/sass_evidence.py)\n")
        f.write("# UBLKCP = cp.async.bulk (TMA 1-D bulk copy), SYNCS = mbarrier ops, LDGSTS = cp.async, REDUX = redux.sync, ATOMS = shared atomics, REDG/ATOMG = global\n")
        f.write("# reductions/atomics, MATCH = match.any, .EF = evict-first (cache-streaming) global accesses, DFMA/DMUL/MUFU.RCP64H = fp64 (shared-reciprocal division)\n")
        f.write("# level kernel <M, warps, entries per lane, update>: the instantiations the BASELINE workloads launch — <7,8,2,2> KDD 5-class, <7,16,1,2> KDD 23-class,\n")
        f.write("# <9,32,1,2> CICIDS 14/15-class, <9,8,2,2> CICIDS 6-class (update 2 = rotated features) — plus <7,8,2,1> (top-group merge variant) and <0,8,2,0> (generic)\n")
        f.write("# kernel | total | " + " | ".join(COLS) + "\n")
        f.write("\n".join(sass()) + "\n")
    with open(os.path.join(ROOT, "profiles", "r02_ptxas_resources.txt"), "w") as f:
        f.write("# ptxas -v resource usage per kernel (nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false), from csrc/build/*.ptxas.log (tools/sass_evidence.py)\n")
        f.write("# kernel | registers | spill stores B | spill loads B | static smem B   (level kernel: only the instantiations the BASELINE workloads launch + the merge variant + the generic one)\n")
        f.write("\n".join(ptxas()) + "\n")
