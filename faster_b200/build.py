"""Builds faster_b200/lib/libfaster_b200.so (CUDA kernels + C ABI + host helpers) for sm_90a (H100) with nvcc.

In-tree build: the .so and its objects are git-ignored build products.  Every source is compiled to its own object (in
parallel, rebuilt only when it or a header changed), then linked.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libfaster_b200.so")
SOURCES = ["fq_kernels.cu", "fq_capi.cu", "fq_pair_capi.cu", "fq_map.cu", "fq_paths.cu", "fq_multi.cu", "fq_host.cpp", "fq_decomp.cpp", "fq_jps.cpp", "fq_jps.cu"]
PUBLIC_HEADER = os.path.join(HERE, "..", "include", "faster_b200.h")
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC,-O3,-Wall"]
LINK_FLAGS = ["-shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a", "-ldl"]


def _headers():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))] + \
           [PUBLIC_HEADER, os.path.abspath(__file__)]


def build(force=False, verbose=False, extra_flags=(), out=None):
    """extra_flags/out: build an experimental variant next to the product library (tuning runs only)."""
    tag = "" if out is None else "_" + os.path.splitext(os.path.basename(out))[0]
    objdir = os.path.join(LIBDIR, "obj" + tag)
    os.makedirs(objdir, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    hdr_t = max(os.path.getmtime(f) for f in _headers())
    target = out or LIB
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src + ".o")
        if force or out is not None or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_t):
            jobs.append([nvcc] + NVCC_FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o])
    if not jobs and os.path.exists(target):
        return target

    def run(cmd):
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    run([nvcc] + LINK_FLAGS + [os.path.join(objdir, src + ".o") for src in SOURCES] + ["-o", target])
    return target


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
