#!/usr/bin/env python
"""Per-kernel SASS opcode counts of the built library (cuobjdump -sass), so that the wgmma / TMA claims can be checked
without disassembling the .so by hand.
    python tools/sass_summary.py herro_b200/libherro_b200.so OUT.txt
Mnemonics on sm_90a: HGMMA = wgmma.mma_async, UTMALDG = cp.async.bulk.tensor (TMA), HMMA = mma.sync, LDSM = ldmatrix,
SYNCS = mbarrier."""
import collections
import re
import subprocess
import sys

KEY = ["HGMMA", "WARPSYNC", "UTMALDG", "UTMASTG", "SYNCS", "HMMA", "LDSM", "LDG", "STG", "LDS",
       "STS", "ATOMS", "ATOMG", "PRMT", "POPC", "SHFL", "BAR", "LOP3", "IMAD", "FFMA", "MUFU"]


def main(lib, dst):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    kern, counts, total = None, collections.OrderedDict(), collections.Counter()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
            counts.setdefault(kern, collections.Counter())
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m and kern:
            op = m.group(1)
            counts[kern][op] += 1
            total[kern] += 1
    with open(dst, "w") as f:
        f.write(f"# cuobjdump -sass {lib}: instructions per kernel and counts of the opcodes that identify the hardware path\n")
        f.write(f"# {'kernel':44s} {'instr':>7s}  " + " ".join(f"{k:>7s}" for k in KEY) + "\n")
        for k, c in counts.items():
            f.write(f"{k[:46]:46s} {total[k]:7d}  " + " ".join(f"{c.get(x, 0):7d}" for x in KEY) + "\n")
    print(open(dst).read())


if __name__ == "__main__":
    main(*sys.argv[1:3])
