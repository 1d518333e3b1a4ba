"""In-tree build of the sm_90a (H100) CUDA library (nvcc cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libctr_b200.so")
CSRC_FEED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc_feed")
LIB_FEED = os.path.join(CSRC_FEED, "libctr_feed.so")          # host-side feeder (g++, no CUDA)


def build(verbose: bool = False, jobs: int | None = None) -> str:
    jobs = jobs or max(2, os.cpu_count() or 2)
    proc = subprocess.run(["make", "-C", CSRC, f"-j{jobs}"], capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        print(proc.stdout)
        print(proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError("building libctr_b200.so failed (see output above)")
    proc = subprocess.run(["make", "-C", CSRC_FEED], capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        print(proc.stdout)
        print(proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError("building libctr_feed.so failed (see output above)")
    return LIB


if __name__ == "__main__":
    print(build(verbose=True))
