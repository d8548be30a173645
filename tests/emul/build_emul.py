"""Build the CPU-emulation library (TEST INFRASTRUCTURE ONLY; see cuda_emul.h)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "_build", "libppsci_b200_emul.so")
SRC = os.path.join(ROOT, "paddlescience_b200", "csrc")


def build(force: bool = False) -> str:
    srcs = [os.path.join(SRC, f) for f in os.listdir(SRC)] + [os.path.join(HERE, "cuda_emul.h"),
                                                              os.path.join(ROOT, "include", "ppsci_b200.h")]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(s) for s in srcs):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cmd = ["g++", "-std=c++17", "-O2", "-DPPSCI_EMUL", "-x", "c++", os.path.join(SRC, "engine.cu"),
           "-I" + HERE, "-I" + os.path.join(ROOT, "include"), "-I" + SRC, "-shared", "-fPIC", "-pthread", "-o", OUT]
    subprocess.run(cmd, check=True)
    return OUT


def build_jet_layouts(force: bool = False) -> str:
    """Host harness of the per-element jet step (jet_layouts.cpp) for tests/test_jet_layouts.py."""
    out = os.path.join(HERE, "_build", "libjet_layouts.so")
    srcs = [os.path.join(HERE, "jet_layouts.cpp"), os.path.join(SRC, "jet_layout.cuh"), os.path.join(SRC, "jet_math.h"),
            os.path.join(ROOT, "include", "ppsci_b200.h")]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(s) for s in srcs):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    # no FMA contraction: both layouts must run exactly the arithmetic the source spells out
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", os.path.join(HERE, "jet_layouts.cpp"),
           "-I" + os.path.join(ROOT, "include"), "-I" + SRC, "-shared", "-fPIC", "-o", out]
    subprocess.run(cmd, check=True)
    return out


if __name__ == "__main__":
    print(build(force=True))
