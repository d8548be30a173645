"""In-tree build of the native library (hand-written CUDA for sm_90a, C-ABI in include/)."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
SRC = os.path.join(PKG, "csrc")
OUT = os.path.join(PKG, "lib", "libppsci_b200.so")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the native library cannot be built")


def sources():
    return sorted(os.path.join(SRC, f) for f in os.listdir(SRC))


def build_native(force: bool = False, verbose: bool = False) -> str:
    out = OUT
    deps = sources() + [os.path.join(ROOT, "include", "ppsci_b200.h")]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = [_nvcc()] + NVCC_FLAGS + ["-I" + os.path.join(ROOT, "include"), "-I" + SRC,
                                    os.path.join(SRC, "engine.cu"), "-o", out]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.run(cmd, check=True)
    return out


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))
