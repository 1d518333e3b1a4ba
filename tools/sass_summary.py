#!/usr/bin/env python
"""Counts the Hopper-specific SASS mnemonics per object of libctr_b200.so (evidence that the tensor-core kernels issue wgmma
(HGMMA) and TMA (UTMALDG) and wait on mbarriers (SYNCS)).  Runs without a GPU:

    python tools/sass_summary.py
"""
from __future__ import annotations

import collections
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "recalgorithm_b200", "csrc")
PATTERNS = [("HGMMA", r"\bHGMMA"), ("WARPGROUP.ARRIVE", r"\bWARPGROUP\.ARRIVE"), ("WARPGROUP.DEPBAR", r"\bWARPGROUP\.DEPBAR"),
            ("UTMALDG", r"\bUTMALDG"), ("UTMASTG", r"\bUTMASTG"), ("UBLKCP", r"\bUBLKCP"),
            ("SYNCS", r"\bSYNCS"), ("LDGSTS", r"\bLDGSTS"), ("HMMA(mma.sync)", r"\bHMMA"),
            ("LDG.E.128", r"\bLDG\.E\S*\.128"), ("STG.E.128", r"\bSTG\.E\S*\.128"), ("RED/ATOM", r"\b(RED|ATOM)G?\.")]


def main():
    objs = sorted(glob.glob(os.path.join(CSRC, "*.o")))
    if not objs:
        sys.exit("no objects: run `python -c 'import __graft_entry__ as g; g.build()'` first")
    print("# SASS mnemonic counts per object (cuobjdump -sass, sm_90a); produced by tools/sass_summary.py")
    print("# columns: " + ", ".join(n for n, _ in PATTERNS))
    for o in objs:
        sass = subprocess.run(["cuobjdump", "-sass", o], capture_output=True, text=True).stdout
        per_kernel = collections.OrderedDict()
        cur = None
        for line in sass.splitlines():
            m = re.search(r"Function : (\S+)", line)
            if m:
                cur = m.group(1)
                per_kernel[cur] = collections.Counter()
                continue
            if cur is None:
                continue
            for name, pat in PATTERNS:
                if re.search(pat, line):
                    per_kernel[cur][name] += 1
        tot = collections.Counter()
        for c in per_kernel.values():
            tot.update(c)
        print(f"\n## {os.path.basename(o)}: {len(per_kernel)} kernels; " + ", ".join(f"{n}={tot[n]}" for n, _ in PATTERNS if tot[n]))
        for k, c in per_kernel.items():
            hot = {n: c[n] for n in ("HGMMA", "WARPGROUP.ARRIVE", "UTMALDG", "UTMASTG", "UBLKCP", "HMMA(mma.sync)") if c[n]}
            if hot:
                dem = subprocess.run(["cu++filt", k], capture_output=True, text=True).stdout.strip() or k
                print(f"   {dem[:150]}: " + ", ".join(f"{n}={v}" for n, v in hot.items()))


if __name__ == "__main__":
    main()
