"""Builds daala_b200/libdaala_b200.so (in-tree) with nvcc for sm_90a (H100).

The library is the product: hand-written CUDA kernels plus the C-ABI layer of
include/daala_b200.h.  nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libdaala_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + [
    "-lineinfo", "-O3", "-std=c++17",
    # double-precision PVQ search must follow the reference's operation order:
    # no FMA contraction, IEEE division and square root (SURVEY.md 7.4.3)
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true",
    "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


# extra nvcc flags for tuning experiments, e.g. DAALA_B200_NVCC_FLAGS="-DDAALA_XFORM_THREADS=64"
FLAGS += os.environ.get("DAALA_B200_NVCC_FLAGS", "").split()


def _deps_mtime():
    m = 0.0
    for d, _, files in os.walk(CSRC):
        for f in files:
            if f.endswith((".cuh", ".h", ".inc")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    m = max(m, os.path.getmtime(os.path.join(ROOT, "include", "daala_b200.h")))
    return m


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdr_m = _deps_mtime()
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m):
            jobs.append([NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    with ThreadPoolExecutor(max_workers=8) as ex:
        logs = list(ex.map(run, jobs))
    if verbose:
        for l in logs:
            sys.stderr.write(l)
    if jobs or not os.path.exists(LIB):
        run([NVCC, "-shared", "-o", LIB] + objs + ARCH)
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
