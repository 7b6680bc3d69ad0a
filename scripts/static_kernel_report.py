#!/usr/bin/env python
"""Static evidence for every kernel of libr2xray.so (no GPU needed): registers / shared memory / spills from
`cuobjdump -res-usage`, and the count of the SASS mnemonics that show what the kernel is built from -- UBLKCP (TMA bulk
copy), LDGSTS (cp.async), SYNCS (mbarrier), MUFU.EX2, FSET / FMNMX, ATOM / RED (atomics),
BAR (barriers) -- from `cuobjdump -sass`.

    python scripts/static_kernel_report.py > profiles/r02_static_kernel_report.txt"""
import os
import re
import subprocess
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "r2_gaussian_b200", "libr2xray.so")
WATCH = ["UBLKCP", "LDGSTS", "SYNCS", "MUFU.EX2", "FSET", "FMNMX", "VOTE", "ATOMS", "ATOMG", "RED",
         "BAR", "ACQBULK", "LDS", "STS", "LDG", "STG"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    res = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            usage[cur] = {k: int(v) for k, v in re.findall(r"(REG|STACK|SHARED|LOCAL|CONSTANT\[0\]):(\d+)", line)}
            cur = None
    sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
    counts, total = {}, {}
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur], total[cur] = Counter(), 0
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if cur and m:
            op = m.group(1)
            total[cur] += 1
            for w in WATCH:
                if op == w or op.startswith(w + ".") or (w == "MUFU.EX2" and op.startswith("MUFU.EX2")):
                    counts[cur][w] += 1
    names = demangle(sorted(usage))
    print(f"# {os.path.relpath(SO, ROOT)}: {len(usage)} kernels, sm_90a; columns: registers, stack bytes, static shared bytes, SASS instructions, watched mnemonics")
    for mangled in sorted(usage, key=lambda k: names[k]):
        u = usage[mangled]
        short = re.sub(r"\(.*", "", names[mangled].replace("(anonymous namespace)::", "")).replace("void ", "")
        c = counts.get(mangled, Counter())
        marks = " ".join(f"{w}={c[w]}" for w in WATCH if c[w])
        print(f"{short:<58} REG={u.get('REG', 0):<3} STACK={u.get('STACK', 0):<4} SHARED={u.get('SHARED', 0):<6} "
              f"SASS={total.get(mangled, 0):<5} {marks}")


if __name__ == "__main__":
    sys.exit(main())
