"""Builds libzqb200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Usage: python zpaqfranz_b200/build.py [--force] [-v]   (run by path: the package itself needs the library)
The built .so is git-ignored; it is rebuilt when a source, a header or this file (the flags) is newer.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("ZQ_LIB", os.path.join(HERE, "libzqb200.so"))   # ZQ_LIB: a tuning build beside the shipped one
SOURCES = ["zq_api.cu", "zq_config.cpp", "zq_cm_host.cpp", "libzpaq_b200.cpp", "zq_archive.cpp", "zq_pipe.cpp", "zq_jit.cpp", "zq_dist.cpp"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-shared", "-cudart", "static",
]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    if os.path.getmtime(os.path.abspath(__file__)) > t:
        return True
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if os.path.getmtime(os.path.join(root, f)) > t:
                return True
    return False


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    extra = os.environ.get("ZQ_EXTRA_FLAGS", "").split()   # tuning builds, e.g. -DZQ_SORT_PROF
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + srcs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
