#!/usr/bin/env python
"""Registers / stack / static shared memory of every kernel in the in-tree objects (cuobjdump --dump-resource-usage), demangled:
the static side of occupancy -- no GPU needed.

    python tools/resource_usage.py
"""
import glob
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return [re.sub(r"\(.*$", "", re.sub(r"^void ", "", n)) for n in out]


def main():
    print("# cuobjdump --dump-resource-usage of recalgorithm_b200/csrc/*.o (sm_90a); produced by tools/resource_usage.py")
    print("# 64 K registers and 64 resident warps per SM: a CTA of W warps at R registers/thread fits floor(65536 / (32*W*ceil8(R))) times")
    for obj in sorted(glob.glob(os.path.join(ROOT, "recalgorithm_b200", "csrc", "*.o"))):
        txt = subprocess.run(["cuobjdump", "--dump-resource-usage", obj], capture_output=True, text=True).stdout
        items = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", txt)
        if not items:
            continue
        print(f"\n## {os.path.basename(obj)}: {len(items)} kernels")
        for name, (_, reg, stack, shared) in sorted(zip(demangle([i[0] for i in items]), items)):
            print(f"   REG {int(reg):3d}  STACK {int(stack):4d}  SHARED(static) {int(shared):6d}   {name[:150]}")


if __name__ == "__main__":
    main()
