"""Build libnts_b200.so (hand-written sm_90a kernels for H100 + C ABI) in-tree with nvcc.

    python -m neutronstarlite_b200.build [--force] [--verbose]

The shared object lands in neutronstarlite_b200/lib/ (git-ignored build product).  nvcc cross-compiles for sm_90a
without a GPU.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIB = os.path.join(LIBDIR, "libnts_b200.so")

CU_SOURCES = ["nts_runtime.cu", "nts_aggregate.cu", "nts_plan.cu", "nts_edge_ops.cu", "nts_exchange.cu", "nts_exchange_plan.cu",
              "nts_graph_build.cu", "nts_sample.cu", "nts_infer.cu", "nts_embedding.cu"]
CXX_SOURCES = ["nts_graph_host.cpp"]
HEADERS = [os.path.join(CSRC, "nts_common.cuh"), os.path.join(ROOT, "include", "nts_b200.h")]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fopenmp",
    "-Xptxas", "-v",
    "-I", os.path.join(ROOT, "include"),
    "-I", CSRC,
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: libnts_b200 cannot be built (there is no CPU fallback)")
    return exe


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd, verbose, log):
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log.append("$ " + " ".join(cmd) + "\n" + res.stdout)
    if verbose:
        print("$ " + " ".join(cmd))
        print(res.stdout)
    if res.returncode != 0:
        raise RuntimeError("build failed:\n$ %s\n%s" % (" ".join(cmd), res.stdout))


def build(force=False, verbose=False):
    """Compile every CUDA/C++ source for sm_90a and link libnts_b200.so. Returns the library path."""
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()
    log = []
    objs = []
    relink = force
    for src in CU_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src + ".o")
        objs.append(o)
        if force or _stale(o, [s] + HEADERS):
            _run([nvcc] + NVCC_FLAGS + ["-c", s, "-o", o], verbose, log)
            relink = True
    for src in CXX_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src + ".o")
        objs.append(o)
        if force or _stale(o, [s] + HEADERS):
            _run(["g++", "-O3", "-std=c++17", "-fPIC", "-fopenmp", "-I", os.path.join(ROOT, "include"),
                  "-c", s, "-o", o], verbose, log)
            relink = True
    if relink or not os.path.exists(LIB):
        _run([nvcc] + ARCH + ["-shared", "-o", LIB] + objs +
             ["-Xcompiler", "-fopenmp", "-lgomp"], verbose, log)
    with open(os.path.join(LIBDIR, "build.log"), "a") as f:
        f.write("\n".join(log))
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or "-v" in sys.argv)
    print(path)
