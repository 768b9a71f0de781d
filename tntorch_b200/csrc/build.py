"""Build libtnb200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python tntorch_b200/csrc/build.py [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "libtnb200.so")
SOURCES = ["tnb200.cu"]
DEPS = [f for f in os.listdir(HERE) if f.endswith((".cu", ".cuh"))] + ["../../include/tnb200.h"]


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(os.path.join(HERE, d)) <= t for d in DEPS)


def build(force=False, verbose=False):
    if not force and up_to_date():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [
        nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
        "-shared", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
        "-I", os.path.join(HERE, "..", "..", "include"),
        "-o", OUT,
    ] + [os.path.join(HERE, s) for s in SOURCES] + ["-lcudart"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
