"""Builds libhyphy_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
from __future__ import annotations

import glob
import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libhyphy_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _newest_input() -> float:
    files = glob.glob(os.path.join(CSRC, "*")) + [os.path.join(os.path.dirname(PKG), "include", "hyphy_b200.h")]
    return max(os.path.getmtime(f) for f in files)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_input():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    for src in sources():
        obj = os.path.join(CSRC, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        subprocess.check_call(cmd)
        objs.append(obj)
    # soname: hosts that link the library (host/Makefile) find it through their rpath, not through the build-time path
    subprocess.check_call([nvcc, "-shared"] + ARCH + ["-Xlinker", "-soname,libhyphy_b200.so",
                           "-o", LIB] + objs + ["-ldl"])
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force=True, verbose="-v" in sys.argv))
