#!/usr/bin/env python
"""SASS instruction counts per kernel of the shipped library (cuobjdump -sass; runs without a GPU): the mnemonics that prove
wgmma / TMA are what the kernels execute, and that no mma.sync (HMMA) path exists.
usage: python tools/sass_summary.py [out.txt]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pretorched_x_b200 import _lib  # noqa: E402

COLS = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "SYNCS", "LDGSTS", "HMMA", "MUFU", "LDS", "STS",
        "LDG", "STG"]


def main():
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", _lib.lib_path()], capture_output=True, text=True).stdout
    names = subprocess.run(["/usr/local/cuda/bin/cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True,
                           text=True).stdout.splitlines()
    counts, order, cur, k = {}, [], None, -1
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            k += 1
            cur = names[k] if k < len(names) else m.group(1)
            cur = re.sub(r"^void ", "", cur).replace("b2::", "").replace("(int)", "").replace("(bool)", "").split("(")[0]
            counts[cur] = collections.Counter()
            order.append(cur)
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            op = m.group(1)
            counts[cur]["total"] += 1
            for c in COLS:
                if op.startswith(c):
                    counts[cur][c] += 1
    out = ["SASS instruction counts per kernel of libb2pretorched.so (cuobjdump -sass, sm_90a): wgmma = HGMMA, wgmma fence / wait = WARPGROUP,",
           "TMA load / store / prefetch = UTMALDG / UTMASTG / UTMAPF, mbarrier = SYNCS,",
           "cp.async = LDGSTS; HMMA (mma.sync) must be 0 everywhere.", "",
           "%-60s" % "kernel" + "".join("%8s" % c for c in COLS) + "%8s" % "total"]
    for name in order:
        c = counts[name]
        out.append("%-60s" % name[:60] + "".join("%8d" % c[x] for x in COLS) + "%8d" % c["total"])
    tot = collections.Counter()
    for c in counts.values():
        tot.update(c)
    out.append("%-60s" % "ALL" + "".join("%8d" % tot[x] for x in COLS) + "%8d" % tot["total"])
    text = "\n".join(out) + "\n"
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
