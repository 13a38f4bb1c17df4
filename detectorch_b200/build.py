"""Builds the sm_90a CUDA library IN-TREE (detectorch_b200/csrc/libdetectorch_b200.so) with nvcc.
The .so is a build product (git-ignored); build() recreates it whenever a CUDA source is newer."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libdetectorch_b200.so")
SOURCES = ["capi_ops.cu", "capi_engine.cu", "capi_coco.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-DNDEBUG"]


STAMP = LIB + ".flags"       # the nvcc command line the library was built with (a library built for another target is rebuilt)


def needs_build():
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != " ".join(NVCC_FLAGS + SOURCES):
            return True
    t = os.path.getmtime(LIB)
    for root, _, files in os.walk(CSRC):
        for f in files:
            if f.endswith((".cu", ".cuh", ".inc", ".h")) and os.path.getmtime(os.path.join(root, f)) > t:
                return True
    hdr = os.path.join(HERE, "..", "include", "detectorch_b200.h")
    return os.path.exists(hdr) and os.path.getmtime(hdr) > t


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    cmd = ["nvcc"] + NVCC_FLAGS + ["-o", LIB] + srcs
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    subprocess.check_call(cmd, cwd=CSRC)
    with open(STAMP, "w") as f:
        f.write(" ".join(NVCC_FLAGS + SOURCES))
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
