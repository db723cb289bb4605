"""Build libpww_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m paint_with_words_sd_b200.csrc.build [--force] [--verbose]

The .so is a build product (git-ignored); the stamp file holds a fingerprint of the sources and flags, so a stale
library is rebuilt.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
LIB = os.path.join(PKG, "libpww_b200.so")
STAMP = os.path.join(PKG, ".libpww_b200.stamp")
SOURCES = ["pww_abi.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _fingerprint() -> str:
    h = hashlib.sha256()
    for root in (HERE, os.path.join(os.path.dirname(PKG), "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == fp:
        return LIB
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB, *[os.path.join(HERE, s) for s in SOURCES]]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libpww_b200.so")
    with open(os.path.join(PKG, "build_ptxas.log"), "w") as f:
        f.write(r.stdout + r.stderr)
    with open(STAMP, "w") as f:
        f.write(fp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
