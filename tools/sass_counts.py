#!/usr/bin/env python
"""SASS evidence: per kernel of libcpi_b200.so the counts of the instructions the design rests on
(UBLKCP = 1-D TMA bulk copy, SYNCS = mbarrier, DFMA/DMUL/DADD = fp64 pipe, FFMA = fp32 variant, SHFL = trio gathers, LDS/STS = slots,
tensor-core opcodes = must be zero).    python tools/sass_counts.py"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = ["UBLKCP", "SYNCS", "DFMA", "DMUL", "DADD", "FFMA", "SHFL", "LDS", "STS", "LDL", "STL", "MUFU", "HMMA", "HGMMA", "BAR"]


def main():
    lib = os.path.join(ROOT, "cpi_b200", "libcpi_b200.so")
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    kern, counts, size = None, collections.OrderedDict(), {}
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            counts[kern] = collections.Counter(); size[kern] = 0
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,5}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", line)
        if m and kern:
            size[kern] += 1
            op = m.group(1)
            for o in OPS:
                if op.startswith(o):
                    counts[kern][o] += 1
    print("# cuobjdump -sass cpi_b200/libcpi_b200.so (sm_90a): static instruction counts per kernel")
    print(f"{'kernel':86s} {'instr':>6s} " + " ".join(f"{o:>6s}" for o in OPS))
    for k, c in counts.items():
        print(f"{k[:86]:86s} {size[k]:6d} " + " ".join(f"{c[o]:6d}" for o in OPS))


if __name__ == "__main__":
    main()
