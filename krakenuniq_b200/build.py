"""Build libkuq.so (the CUDA extension) in-tree with nvcc for sm_90a (H100).  The .so is a build product and
stays out of git."""
from __future__ import annotations

import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "lib", "libkuq.so")
SOURCES = ["kuq_kernels.cu", "kuq_api.cu", "kuq_dbbuild.cu", "kuq_microbench.cu", "kuq_layout_exp.cu", "kuq_clades.cu",
           "kuq_collisions.cu", "kuq_kmerset.cu", "kuq_countunique.cu"]
HEADERS = ["kuq_kernels.cuh", "kuq_buffers.cuh", "kuq_minimizer.cuh", "kuq_bounce.cuh", "kuq_ranges.h", "kuq_batches.h",
           "kuq_kmerpack.cuh", "kuq_dbfile.h",
           os.path.join(ROOT, "include", "kuq.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--compiler-bindir", "/usr/bin/g++", "-Xcompiler", "-fPIC,-O2,-Wall", "-shared", "-cudart", "shared"]


def nvcc():
    for c in (os.environ.get("KUQ_NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libkuq.so")
    if verbose:
        sys.stderr.write(r.stderr)
    return LIB


CLASSIFY = os.path.join(PKG, "bin", "classify")


def build_classify(force: bool = False) -> str:
    """The drop-in `classify` executable (host C++ over libkuq.so) and, from the same source with -DEXACT_COUNTING
    like the reference's Makefile, `classifyExact` (what `krakenuniq --exact` runs)."""
    src = os.path.join(CSRC, "classify_main.cpp")
    build(force=force)
    exact = CLASSIFY + "Exact"
    newest = max(os.path.getmtime(p) for p in [src, LIB] + [os.path.join(CSRC, h) for h in ("kuq_batches.h", "kuq_ranges.h", "kuq_dbfile.h")])
    if not force and all(os.path.exists(x) and os.path.getmtime(x) >= newest for x in (CLASSIFY, exact)):
        return CLASSIFY
    os.makedirs(os.path.dirname(CLASSIFY), exist_ok=True)
    for out, defs in ((CLASSIFY, []), (exact, ["-DEXACT_COUNTING"])):
        cmd = ["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-fopenmp"] + defs + [src, "-o", out, "-L" + os.path.dirname(LIB),
               "-lkuq", "-lz", "-ldl", "-Wl,-rpath,$ORIGIN/../lib", "-Wl,-rpath,/usr/local/cuda/lib64"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("g++ failed building " + os.path.basename(out))
    return CLASSIFY


KMER_SET = os.path.join(PKG, "bin", "kmer_set")
COUNT_UNIQUE = os.path.join(PKG, "bin", "count_unique")


def build_dbtools(force: bool = False):
    """The drop-in `db_sort` and `set_lcas` executables (SURVEY §8 f4; host C++ over libkuq.so), `kmer_set`, the
    drop-in for build_db.sh's Jellyfish 1 step (at KMER_SET), and `count_unique` (at COUNT_UNIQUE).  Returns the paths
    of db_sort and set_lcas."""
    src = os.path.join(CSRC, "dbbuild_main.cpp")
    build(force=force)
    outs = [(os.path.join(PKG, "bin", "db_sort"), src, [], []),
            (os.path.join(PKG, "bin", "set_lcas"), src, ["-DTOOL_SET_LCAS"], []),
            (KMER_SET, os.path.join(CSRC, "kmerset_main.cpp"), [], []),
            (COUNT_UNIQUE, os.path.join(CSRC, "countunique_main.cpp"), [], ["-lz"])]
    newest = max([os.path.getmtime(s) for _, s, _, _ in outs] + [os.path.getmtime(LIB)] +
                 [os.path.getmtime(os.path.join(CSRC, h)) for h in ("kuq_ranges.h", "kuq_dbfile.h")])
    if not force and all(os.path.exists(o) and os.path.getmtime(o) >= newest for o, _, _, _ in outs):
        return [o for o, _, _, _ in outs[:2]]
    os.makedirs(os.path.join(PKG, "bin"), exist_ok=True)
    for out, src, defs, libs in outs:
        cmd = ["/usr/bin/g++", "-O2", "-std=c++17", "-Wall"] + defs + [src, "-o", out, "-L" + os.path.dirname(LIB), "-lkuq"] + \
              libs + ["-Wl,-rpath,$ORIGIN/../lib", "-Wl,-rpath,/usr/local/cuda/lib64"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("g++ failed building " + os.path.basename(out))
    return [o for o, _, _, _ in outs[:2]]


if __name__ == "__main__":
    build_dbtools(force="--force" in sys.argv)
    build_classify(force="--force" in sys.argv)
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
