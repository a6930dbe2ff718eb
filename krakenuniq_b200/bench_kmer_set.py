"""Throughput of `kmer_set` (step 1 of build_db.sh on the GPU) on a seeded synthetic library; prints one JSON line.

The library: `--gbp` Gbp in `--strains` mutated copies (0.1 % substitutions) of random genomes, 1 Mbp records in
80-column FASTA, so that the k-mer set is about a seventh of the windows, as in a library of related strains.
Measured:
  - file → PREFIX_0: the executable end to end (parse, pack, passes, writing the file), Gbp / wall second;
  - packed: the passes alone through the C ABI once the library sits packed in HBM (kuq_kmer_set_next until the end),
    Gbp / second; per-stage device times from kuq_kmer_set_stats; the executable's own parse time;
  - the same with an HBM budget that forces several passes.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_kmer_set.py [--gbp 2] [--k 31]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import binding, build  # noqa: E402

RECORD = 1_000_000
WIDTH = 80


def make_library(path, gbp, strains, seed):
    """writes the FASTA; returns (bases u8, offsets u64) of the same records for the C ABI"""
    rng = np.random.default_rng(seed)
    total = int(gbp * 1e9) // (strains * RECORD) * (strains * RECORD)
    base = rng.integers(0, 4, total // strains, dtype=np.uint8)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    bases = np.empty(total, np.uint8)
    for s in range(strains):
        c = base.copy()
        m = rng.integers(0, len(c), len(c) // 1000)
        c[m] = (c[m] + rng.integers(1, 4, len(m), dtype=np.uint8)) & 3
        bases[s * len(c):(s + 1) * len(c)] = acgt[c]
    with open(path, "wb") as f:
        for r in range(total // RECORD):
            seq = bases[r * RECORD:(r + 1) * RECORD].reshape(-1, WIDTH)
            f.write(b">r%d strain %d\n" % (r, r * RECORD // len(base)))
            f.write(np.hstack([seq, np.full((len(seq), 1), ord("\n"), np.uint8)]).tobytes())
    return bases, np.arange(0, total + 1, RECORD, dtype=np.uint64)


def drain(ks, buf):
    t = time.perf_counter()
    while ks.next(buf):
        pass
    return time.perf_counter() - t


def packed_run(bases, offs, k, budget=None):
    ks = binding.KmerSet(k, budget)
    t = time.perf_counter()
    ks.add(bases, offs)
    ks.info()                                    # waits for the packing and plans the passes
    add_s = time.perf_counter() - t
    next_s = drain(ks, np.zeros((1 << 22) * ks.rec, np.uint8))
    key_ct, passes = ks.info()
    st = ks.stats()
    ks.close()
    gbp = len(bases) / 1e9
    return {"passes": passes, "distinct_kmers": key_ct, "add_s": round(add_s, 3), "passes_s": round(next_s, 3),
            "packed_gbp_per_s": round(gbp / next_s, 3), "stage_ms": {a: round(b, 2) for a, b in st["stage_ms"].items()},
            "windows": st["windows"], "library_in_hbm": st["library_in_hbm"],
            "planned_bytes": st["ws_estimate_bytes"], "measured_peak_bytes": st["peak_bytes"]}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                       # the numbers still stand; say what is missing
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=2.0)
    ap.add_argument("--k", type=int, default=31)
    ap.add_argument("--strains", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--passes", type=int, default=6, help="passes the forced multi-pass run aims at")
    a = ap.parse_args()
    build.build_dbtools()
    tmp = tempfile.mkdtemp(prefix="kuq_kmer_set_")
    try:
        lib = os.path.join(tmp, "lib.fa")
        t = time.perf_counter()
        bases, offs = make_library(lib, a.gbp, a.strains, a.seed)
        gen_s = time.perf_counter() - t
        gbp = len(bases) / 1e9
        packed_run(bases[:1 << 24], offs[:17], a.k)                    # warm-up: module load, CUB's first launches
        cmd = [build.KMER_SET, "count", "-m", str(a.k), "-s", "1G", "-C", "-t", "8", "-o", os.path.join(tmp, "database"), lib]
        subprocess.run(cmd, check=True, capture_output=True)           # warm the page cache and the driver
        os.remove(os.path.join(tmp, "database_0"))
        t = time.perf_counter()
        r = subprocess.run(cmd, check=True, capture_output=True, text=True)
        file_s = time.perf_counter() - t
        out_bytes = os.path.getsize(os.path.join(tmp, "database_0"))
        os.remove(os.path.join(tmp, "database_0"))
        summary = r.stderr.strip().splitlines()[-1]
        parse_s = float(summary.split("of which parsing ")[1].split(" s")[0])
        one = packed_run(bases, offs, a.k)
        budget = one["planned_bytes"] // a.passes + (8 << 20)
        multi = packed_run(bases, offs, a.k, budget)
        multi["budget_bytes"] = budget
        print(json.dumps({"metric": "kmer_set", "k": a.k, "gbp": round(gbp, 3), "gpu": gpu_info(),
                          "file_to_prefix0_gbp_per_s": round(gbp / file_s, 3), "file_to_prefix0_s": round(file_s, 3),
                          "output_bytes": out_bytes, "host_parse_s": parse_s, "executable_summary": summary,
                          "single": one, "forced_multipass": multi, "library_generation_s": round(gen_s, 1)}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
