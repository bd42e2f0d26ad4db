"""Builds liborbfe.so (hand-written sm_90a CUDA for H100 + the C-ABI) in-tree with nvcc.

No torch, no JIT cache: the .so lands next to this file so that it travels to the GPU box with the
repo snapshot.  nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "liborbfe.so")
SOURCES = ["orbfe_api.cu", "extract_kernels.cu", "match_kernels.cu", "bow_kernels.cu", "kfdb.cu", "comm.cu",
           os.path.join("..", "host", "match_host.cpp"), os.path.join("..", "host", "bow_host.cpp")]
DEPS = SOURCES + ["orbfe_internal.h", "bow_l1.cuh", os.path.join("..", "..", "include", "orbfe.h"),
                  os.path.join("..", "..", "include", "orbfe_match.h"), os.path.join("..", "..", "include", "orbfe_bow.h"), os.path.join("..", "..", "include", "orbfe_comm.h"),
                  os.path.join("..", "..", "include", "orbfe_brief_pattern.inc"), os.path.join("..", "build.py")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",                       # float ops on the device are individually rounded (parity)
    "-Xcompiler", "-fPIC,-ffp-contract=off,-O2",
    "-cudart", "static",
    "-shared",
    "-ldl",
]


def nvcc_path():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if p and (os.path.isabs(p) and os.path.exists(p) or not os.path.isabs(p)):
            return p
    return "nvcc"


def is_stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


E2E_SRC = os.path.join(HERE, "..", "tools", "e2e_driver.cpp")
E2E_SO = os.path.join(HERE, "libe2e_driver.so")


def build_e2e_driver(force=False):
    """bench.py's end-to-end stream pipeline on C++ threads (tools/e2e_driver.cpp): bench harness over the public C-ABI,
    not part of liborbfe.so; plain g++, no CUDA."""
    if not force and os.path.exists(E2E_SO) and os.path.getmtime(E2E_SO) >= max(
            os.path.getmtime(E2E_SRC), os.path.getmtime(os.path.join(HERE, "..", "include", "orbfe_match.h"))):
        return E2E_SO
    cmd = ["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-ffp-contract=off", "-pthread", "-I", os.path.join(HERE, "..", "include"),
           E2E_SRC, "-o", E2E_SO]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("g++ failed building libe2e_driver.so")
    return E2E_SO


def build_native(force=False, verbose=False):
    build_e2e_driver(force)
    if not force and not is_stale():
        return SO
    extra = os.environ.get("ORBFE_NVCC_EXTRA", "").split()   # experiments, e.g. -Xptxas -warn-spills
    cmd = [nvcc_path()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", SO] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed building liborbfe.so")
    if verbose:
        print(r.stdout)
    return SO


if __name__ == "__main__":
    build_native(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(SO)
