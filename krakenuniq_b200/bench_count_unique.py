"""Throughput of `count_unique` (krakenuniq-build's distinct k-mer estimate, on the GPU) on a seeded synthetic library;
prints one JSON line.

The library is shaped like bench_kmer_set.py's: `--gbp` Gbp in `--strains` mutated copies (0.1 % substitutions) of
random genomes, 1 Mbp records in 80-column FASTA.  Measured:
  - the executable end to end, stdin from the file and from a pipe (`cat lib.fa |`), Gbp / wall second, and its own
    parse time (KUQ_COUNT_UNIQUE_STATS);
  - the sketch kernel's device time per Gbp from CUDA events (kuq_count_unique_stats), at p = 14 and p = 18, with the
    library fed through the C ABI;
  - the reference's `count_unique -t 8` (fewer threads on a smaller host) from oracle/_ref/ on the same file, when that
    was built;
  - the card's name, power limit and maximum SM clock.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_count_unique.py [--gbp 2] [--k 31]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import binding, build  # noqa: E402
from krakenuniq_b200.bench_kmer_set import gpu_info, make_library  # noqa: E402


def timed(cmd, stdin_path=None, shell=False, env=None):
    t = time.perf_counter()
    if shell:
        r = subprocess.run(cmd, shell=True, check=True, capture_output=True, text=True, env=env)
    else:
        with open(stdin_path, "rb") as f:
            r = subprocess.run(cmd, stdin=f, check=True, capture_output=True, text=True, env=env)
    return time.perf_counter() - t, r


def kernel_ms_per_gbp(bases, offs, k, p):
    cu = binding.CountUnique(k, p)
    try:
        cu.add(bases, offs)
        est, n, _ = cu.result()
        st = cu.stats()
    finally:
        cu.close()
    return {"estimate": est, "windows": n, "sketch_ms": round(st["sketch_ms"], 3),
            "sketch_ms_per_gbp": round(st["sketch_ms"] / (st["bases"] / 1e9), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=2.0)
    ap.add_argument("--k", type=int, default=31)
    ap.add_argument("--strains", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    build.build_dbtools()
    tmp = tempfile.mkdtemp(prefix="kuq_count_unique_")
    try:
        lib = os.path.join(tmp, "lib.fa")
        bases, offs = make_library(lib, a.gbp, a.strains, a.seed)
        gbp = len(bases) / 1e9
        kernel_ms_per_gbp(bases[:1 << 24], offs[:17], a.k, 14)          # warm-up: module load, first launches
        cmd = [build.COUNT_UNIQUE, "-k", str(a.k)]
        env = dict(os.environ, KUQ_COUNT_UNIQUE_STATS="1")
        timed(cmd, lib)                                                  # warm the page cache and the driver
        file_s, r = timed(cmd, lib, env=env)
        summary = r.stderr.strip().splitlines()[-1]
        parse_s = float(summary.split("(parsing ")[1].split(" s")[0])
        pipe_s, rp = timed(f"cat {lib} | {' '.join(cmd)}", shell=True)
        assert rp.stdout == r.stdout
        out = {"metric": "count_unique", "k": a.k, "gbp": round(gbp, 3), "gpu": gpu_info(), "estimate": int(r.stdout),
               "file_gbp_per_s": round(gbp / file_s, 3), "file_s": round(file_s, 3),
               "pipe_gbp_per_s": round(gbp / pipe_s, 3), "pipe_s": round(pipe_s, 3), "host_parse_s": round(parse_s, 3),
               "executable_summary": summary,
               "kernel_p14": kernel_ms_per_gbp(bases, offs, a.k, 14), "kernel_p18": kernel_ms_per_gbp(bases, offs, a.k, 18)}
        ref = os.path.join(ROOT, "oracle", "_ref", "count_unique")
        if os.path.exists(ref):
            threads = min(8, len(os.sched_getaffinity(0)))
            ref_s, rr = timed([ref, "-k", str(a.k), "-t", str(threads)], lib)
            out["reference_threads"] = threads
            out["reference_gbp_per_s"] = round(gbp / ref_s, 3)
            out["reference_s"] = round(ref_s, 3)
            out["reference_estimate_equal"] = rr.stdout == r.stdout
        else:
            out["reference_gbp_per_s"] = "not measured (oracle/_ref/count_unique not built)"
        print(json.dumps(out))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
