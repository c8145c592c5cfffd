"""Builds finitestateentropy_b200/libfse_b200.so (hand-written sm_90a kernels + the C-ABI) in-tree with nvcc.

nvcc cross-compiles without a GPU; the .so is a build product (git-ignored).  Also builds the two CPU checkers under oracle/ (test infrastructure)."""
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libfse_b200.so")
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--shared", "-cudart", "static",
              "-Xlinker", "-z,defs"]   # an undefined symbol (a launcher declared unlike its definition) fails the link, not the load


def lib_is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    srcs = glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + \
        glob.glob(os.path.join(ROOT, "include", "*.h"))
    return any(os.path.getmtime(s) > t for s in srcs)


def build_lib(force=False, verbose=False):
    if not force and not lib_is_stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-I", os.path.join(ROOT, "include"), "-o", LIB] + srcs
    subprocess.check_call(cmd)
    return LIB


def build_oracles():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "fuzzers"])   # the reference's fuzzers linked against OUR library
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "cli"])       # the reference's file tool (frame-format checker)


def build_programs():
    """host programs over the C-ABI (programs/Makefile): bench_gpu, fse_b200_file"""
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "programs"), "all"])


if __name__ == "__main__":
    import sys
    build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
